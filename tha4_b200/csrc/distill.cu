// Distillation inner loop for the body student (SURVEY.md section 8 a16): SirenMorpher03 forward with stored
// activations, the four L1 loss terms against the teacher, the full backward pass (grid_sample w.r.t. its grid,
// alpha blend, 1x1 layers through sin(30 z), bilinear x2 level hand-offs) into a flat gradient buffer, and Adam.
// Reference: siren_morpher_protocols_03.py:102-157,178-214; siren_morpher_03_trainer.py:32-50 (loss terms);
// siren_morpher_03.py:107-139 (forward); shion/base/loss/l1_loss.py:9-24 (mean |a-b|); optimizer_factories.py:9-17.
//
// Layout: parameters / gradients / Adam moments are flat fp32 buffers in the reference's state_dict order
// (siren_layers.l.j.linear.{weight,bias} ..., last_linear.{weight,bias}); activations are fp32 NHWC with channel
// counts padded to multiples of 4 (360, 180, 92; level inputs 48 / 228 / 140), pad channels are exactly zero.
// The dense layers are GEMMs over all pixels of the micro-batch and run on the same wgmma conv kernel as the
// teacher (1x1 taps); weight gradients use a dedicated pixel-reduction GEMM (mma.sync TF32).
#include "distill.cuh"
#include "gridsample.cuh"
#include "profiler.cuh"

namespace tha4 {
namespace {

constexpr float OMEGA = 30.0f;

// ---------------------------------------------------------------------------------------------- small kernels
// level input: [up(prev) (Cprev, from `prev` at R/2) | x | y | pose(45) | 0 pad]
__global__ void __launch_bounds__(256) level_input_kernel(const float* __restrict__ prev, int Cprev, int prev_ld,
                                                          const float* __restrict__ pose, int pose_ld,
                                                          const float* __restrict__ base, int R, int N, int C, int npose, float* __restrict__ out) {
    const long total = (long)N * R * R * C;
    const int Rh = R >> 1;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int c = (int)(i % C);
        long p = i / C;
        const int x = (int)(p % R); p /= R;
        const int y = (int)(p % R);
        const int n = (int)(p / R);
        float v = 0.0f;
        if (c < Cprev) {
            const LerpTap ty = lerp_locate(y, 0.5f, Rh), tx = lerp_locate(x, 0.5f, Rh);
            const float* pp = prev + (long)n * Rh * Rh * prev_ld + c;
            const float a = pp[((long)ty.i0 * Rh + tx.i0) * prev_ld], b = pp[((long)ty.i0 * Rh + tx.i1) * prev_ld];
            const float cc = pp[((long)ty.i1 * Rh + tx.i0) * prev_ld], d = pp[((long)ty.i1 * Rh + tx.i1) * prev_ld];
            v = ty.l0 * (tx.l0 * a + tx.l1 * b) + ty.l1 * (tx.l0 * cc + tx.l1 * d);
        } else if (c == Cprev) v = base[x];
        else if (c == Cprev + 1) v = base[y];
        else if (c < Cprev + 2 + npose) v = pose[(long)n * pose_ld + (c - Cprev - 2)];
        out[i] = v;
    }
}

// adjoint of the bilinear x2 upsample: dprev[n, j] += sum over the high-res pixels whose taps touch j (gather form)
__global__ void __launch_bounds__(256) upsample_backward_kernel(const float* __restrict__ dup, int up_ld, int Cprev, int R, int N,
                                                                float* __restrict__ dprev, int prev_ld) {
    const int Rh = R >> 1;
    const long total = (long)N * Rh * Rh * Cprev;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int c = (int)(i % Cprev);
        long p = i / Cprev;
        const int jx = (int)(p % Rh); p /= Rh;
        const int jy = (int)(p % Rh);
        const int n = (int)(p / Rh);
        float acc = 0.0f;
        for (int dy = 2 * jy - 2; dy <= 2 * jy + 3; ++dy) {
            if (dy < 0 || dy >= R) continue;
            const LerpTap ty = lerp_locate(dy, 0.5f, Rh);
            const float wy = (ty.i0 == jy ? ty.l0 : 0.0f) + (ty.i1 == jy ? ty.l1 : 0.0f);
            if (wy == 0.0f) continue;
            for (int dx = 2 * jx - 2; dx <= 2 * jx + 3; ++dx) {
                if (dx < 0 || dx >= R) continue;
                const LerpTap tx = lerp_locate(dx, 0.5f, Rh);
                const float wx = (tx.i0 == jx ? tx.l0 : 0.0f) + (tx.i1 == jx ? tx.l1 : 0.0f);
                if (wx == 0.0f) continue;
                acc += wy * wx * dup[(((long)n * R + dy) * R + dx) * up_ld + c];
            }
        }
        dprev[(((long)n * Rh + jy) * Rh + jx) * prev_ld + c] = acc;
    }
}

// a = sin(30 z)   (z, a: [rows][C] contiguous)
__global__ void __launch_bounds__(256) sine_forward_kernel(const float* __restrict__ z, float* __restrict__ a, long n4) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n4; i += (long)gridDim.x * blockDim.x) {
        const float4 v = reinterpret_cast<const float4*>(z)[i];
        reinterpret_cast<float4*>(a)[i] = make_float4(sinf(OMEGA * v.x), sinf(OMEGA * v.y), sinf(OMEGA * v.z), sinf(OMEGA * v.w));
    }
}
// dz = da * 30 cos(30 z)   (in place on da)
__global__ void __launch_bounds__(256) sine_backward_kernel(const float* __restrict__ z, float* __restrict__ da, long n4) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n4; i += (long)gridDim.x * blockDim.x) {
        const float4 v = reinterpret_cast<const float4*>(z)[i];
        float4 g = reinterpret_cast<float4*>(da)[i];
        g.x *= OMEGA * cosf(OMEGA * v.x); g.y *= OMEGA * cosf(OMEGA * v.y);
        g.z *= OMEGA * cosf(OMEGA * v.z); g.w *= OMEGA * cosf(OMEGA * v.w);
        reinterpret_cast<float4*>(da)[i] = g;
    }
}

// db[c] += sum_rows dz[row][c]     (C <= 1024, C % 4 == 0; only the first creal channels are accumulated)
__global__ void __launch_bounds__(256) colsum_kernel(const float* __restrict__ dz, long rows, int C, int creal, float* __restrict__ db) {
    __shared__ float red[256][5];
    const int cq = C >> 2, PL = 256 / cq;
    const int tid = threadIdx.x, pl = tid / cq, q = tid - pl * cq;
    float s[4] = {0, 0, 0, 0};
    if (pl < PL) {
        for (long r = (long)blockIdx.x * PL + pl; r < rows; r += (long)gridDim.x * PL) {
            const float4 v = *reinterpret_cast<const float4*>(dz + r * C + 4 * q);
            s[0] += v.x; s[1] += v.y; s[2] += v.z; s[3] += v.w;
        }
    }
    for (int k = 0; k < 4; ++k) red[tid][k] = s[k];
    __syncthreads();
    if (pl == 0 && pl < PL) {
        float acc[4] = {0, 0, 0, 0};
        for (int j = 0; j < PL; ++j) for (int k = 0; k < 4; ++k) acc[k] += red[j * cq + q][k];
        for (int k = 0; k < 4; ++k) if (4 * q + k < creal) atomicAdd(db + 4 * q + k, acc[k]);
    }
}

// dW[n][k] += sum_p dz[p][n] * x[p][k]   (dz: [P][Nc], x: [P][Kc]; only n < nreal, k < kreal are accumulated into
// dW[nreal][kreal]).  grid = (ceil(Nc/64), ceil(Kc/64), P-splits); 128 threads = 2x2 warps of 32x32; TF32 mma.sync.
__device__ __forceinline__ unsigned f2tf32(float f) { unsigned r; asm("cvt.rna.tf32.f32 %0, %1;\n" : "=r"(r) : "f"(f)); return r; }
__device__ __forceinline__ void mma8(float (&c)[4], const unsigned (&a)[4], unsigned b0, unsigned b1) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
constexpr int WG_P = 32, WG_PITCH = 72;
__global__ void __launch_bounds__(128) wgrad_kernel(const float* __restrict__ dz, int Nc, const float* __restrict__ x, int Kc,
                                                    long P, int nreal, int kreal, float* __restrict__ dW) {
    __shared__ __align__(16) float sd[WG_P][WG_PITCH];
    __shared__ __align__(16) float sx[WG_P][WG_PITCH];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, t = lane & 3;
    const int wm = warp & 1, wn = warp >> 1;
    const int n0 = blockIdx.x * 64, k0 = blockIdx.y * 64;
    const long per = (P + gridDim.z - 1) / gridDim.z;
    const long pb = blockIdx.z * per, pe = min(P, pb + per);
    float acc[2][4][4];
    for (int i = 0; i < 2; ++i) for (int j = 0; j < 4; ++j) for (int k = 0; k < 4; ++k) acc[i][j][k] = 0.0f;
    for (long p0 = pb; p0 < pe; p0 += WG_P) {
        // stage 32 pixels x 64 columns of dz and x (zero beyond the matrix / pixel range)
        for (int i = tid; i < WG_P * 16; i += 128) {
            const int r = i >> 4, q = i & 15;
            const long p = p0 + r;
            float4 vd = make_float4(0.f, 0.f, 0.f, 0.f), vx = vd;
            if (p < pe) {
                if (n0 + 4 * q < Nc) vd = *reinterpret_cast<const float4*>(dz + p * Nc + n0 + 4 * q);
                if (k0 + 4 * q < Kc) vx = *reinterpret_cast<const float4*>(x + p * Kc + k0 + 4 * q);
            }
            *reinterpret_cast<float4*>(&sd[r][4 * q]) = vd;
            *reinterpret_cast<float4*>(&sx[r][4 * q]) = vx;
        }
        __syncthreads();
#pragma unroll
        for (int ks = 0; ks < WG_P / 8; ++ks) {
            unsigned a[2][4];
#pragma unroll
            for (int mt = 0; mt < 2; ++mt) {           // A[m = n index][k = pixel] = dz[pixel][n]
                const int m = wm * 32 + mt * 16 + g;
                a[mt][0] = f2tf32(sd[ks * 8 + t][m]);
                a[mt][1] = f2tf32(sd[ks * 8 + t][m + 8]);
                a[mt][2] = f2tf32(sd[ks * 8 + t + 4][m]);
                a[mt][3] = f2tf32(sd[ks * 8 + t + 4][m + 8]);
            }
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {           // B[k = pixel][n = k index] = x[pixel][k]
                const int c = wn * 32 + nt * 8 + g;
                const unsigned b0 = f2tf32(sx[ks * 8 + t][c]), b1 = f2tf32(sx[ks * 8 + t + 4][c]);
                mma8(acc[0][nt], a[0], b0, b1);
                mma8(acc[1][nt], a[1], b0, b1);
            }
        }
        __syncthreads();
    }
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int n = n0 + wm * 32 + mt * 16 + g + h * 8;
                const int k = k0 + wn * 32 + nt * 8 + 2 * t;
                if (n < nreal) {
                    if (k < kreal) atomicAdd(dW + (long)n * kreal + k, acc[mt][nt][2 * h]);
                    if (k + 1 < kreal) atomicAdd(dW + (long)n * kreal + k + 1, acc[mt][nt][2 * h + 1]);
                }
            }
}

// packed[co][ci] (conv layout, zero padded) = W[co][ci] or its transpose
__global__ void pack_dense_kernel(const float* __restrict__ W, int nreal, int kreal, int transpose, float* __restrict__ dst,
                                  int cout_pad, int cin_pad) {
    const int total = cout_pad * cin_pad;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const int co = i / cin_pad, ci = i - co * cin_pad;
        float v = 0.0f;
        if (!transpose) { if (co < nreal && ci < kreal) v = W[(long)co * kreal + ci]; }
        else { if (co < kreal && ci < nreal) v = W[(long)ci * kreal + co]; }
        dst[i] = round_tf32(v);
    }
}
__global__ void pad_bias_kernel(const float* __restrict__ b, int nreal, int npad, float* __restrict__ dst) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < npad) dst[i] = i < nreal ? b[i] : 0.0f;
}

// Bilinear sample of one pixel at base + grid change (the arithmetic of gridsample.cuh), with what its backward needs.
// mx / my: d(ix)/d(grid_x), d(iy)/d(grid_y) = R/2 inside the image, 0 where the border clamp is active (ATen
// clip_coordinates_set_grad).  Out-of-range corners read as 0.
struct SampleAt {
    int x0, y0;
    bool xin, yin;
    float tx, ty, mx, my;
};
__device__ __forceinline__ SampleAt sample_locate(const float* __restrict__ base, int x, int y, float gcx, float gcy, int R) {
    SampleAt s;
    const float ixu = __fdiv_rn(__fsub_rn(__fmul_rn(__fadd_rn(__fadd_rn(base[x], gcx), 1.0f), (float)R), 1.0f), 2.0f);
    const float iyu = __fdiv_rn(__fsub_rn(__fmul_rn(__fadd_rn(__fadd_rn(base[y], gcy), 1.0f), (float)R), 1.0f), 2.0f);
    const float ix = fminf((float)(R - 1), fmaxf(ixu, 0.0f)), iy = fminf((float)(R - 1), fmaxf(iyu, 0.0f));
    s.mx = (ixu <= 0.0f || ixu >= (float)(R - 1)) ? 0.0f : 0.5f * R;
    s.my = (iyu <= 0.0f || iyu >= (float)(R - 1)) ? 0.0f : 0.5f * R;
    const float fx = floorf(ix), fy = floorf(iy);
    s.x0 = (int)fx; s.y0 = (int)fy;
    s.xin = s.x0 + 1 < R; s.yin = s.y0 + 1 < R;
    s.tx = ix - fx; s.ty = iy - fy;
    return s;
}
// the four corners of one channel plane `im` (row stride sh), the sampled value and its derivatives w.r.t. ix and iy
struct Corners { float v00, v01, v10, v11; };
__device__ __forceinline__ Corners sample_corners(const float* im, long sh, const SampleAt& s) {
    Corners v;
    v.v00 = im[(long)s.y0 * sh + s.x0];
    v.v01 = s.xin ? im[(long)s.y0 * sh + s.x0 + 1] : 0.0f;
    v.v10 = s.yin ? im[(long)(s.y0 + 1) * sh + s.x0] : 0.0f;
    v.v11 = (s.xin && s.yin) ? im[(long)(s.y0 + 1) * sh + s.x0 + 1] : 0.0f;
    return v;
}
__device__ __forceinline__ float sample_value(const Corners& v, const SampleAt& s) {
    return (v.v00 * (1.0f - s.tx) + v.v01 * s.tx) * (1.0f - s.ty) + (v.v10 * (1.0f - s.tx) + v.v11 * s.tx) * s.ty;
}
__device__ __forceinline__ float sample_dix(const Corners& v, const SampleAt& s) {
    return (v.v01 - v.v00) * (1.0f - s.ty) + (v.v11 - v.v10) * s.ty;
}
__device__ __forceinline__ float sample_diy(const Corners& v, const SampleAt& s) {
    return (v.v10 - v.v00) * (1.0f - s.tx) + (v.v11 - v.v01) * s.tx;
}

// Fused tail: forward of grid_sample + blend, the four L1 terms, and the gradient w.r.t. the head output.
// out7: [P][8] = grid_change(0,1) alpha(2) colour(3..6) pad; image / targets NCHW.  d_out7: [P][8].
// loss_acc: doubles [4] = sum|blended-T0|, sum|warped-T2|, sum|grid-T3|, sum|colour-T0|.
// wn[4]: weight_i / element count of term i (mean reduction, l1_loss.py:19-21).
__device__ __forceinline__ float sgn(float v) { return v > 0.0f ? 1.0f : (v < 0.0f ? -1.0f : 0.0f); }
__global__ void __launch_bounds__(256) train_tail_kernel(const float* __restrict__ out7, ImgView image, const float* __restrict__ T0,
                                                         const float* __restrict__ T2, const float* __restrict__ T3,
                                                         const float* __restrict__ base, int R, float4 wn,
                                                         float* __restrict__ d_out7, double* __restrict__ loss_acc) {
    __shared__ float red[8][4];
    const long hw = (long)R * R, total = image.N * hw;
    float l[4] = {0, 0, 0, 0};
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int x = (int)(i % R), y = (int)((i / R) % R), n = (int)(i / hw);
        const long pp = (long)y * R + x;
        const float4 oa = *reinterpret_cast<const float4*>(out7 + i * 8), ob = *reinterpret_cast<const float4*>(out7 + i * 8 + 4);
        const float gcx = oa.x, gcy = oa.y, alpha = oa.z;
        const float col[4] = {oa.w, ob.x, ob.y, ob.z};
        const SampleAt sa = sample_locate(base, x, y, gcx, gcy, R);
        const float mx = sa.mx, my = sa.my;
        float gix = 0.0f, giy = 0.0f, dalpha = 0.0f, dcol[4];
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            const Corners v = sample_corners(image.p + n * image.sn + c * image.sc, image.sh, sa);
            const float wp = sample_value(v, sa);
            const float bl = (1.0f - alpha) * wp + alpha * col[c];
            const long ti = ((long)n * 4 + c) * hw + pp;
            const float t0 = T0[ti], t2 = T2[ti];
            l[0] += fabsf(bl - t0); l[1] += fabsf(wp - t2); l[3] += fabsf(col[c] - t0);
            const float dbl = wn.x * sgn(bl - t0);
            const float dwp = dbl * (1.0f - alpha) + wn.y * sgn(wp - t2);
            dalpha += dbl * (col[c] - wp);
            dcol[c] = dbl * alpha + wn.w * sgn(col[c] - t0);
            gix += dwp * sample_dix(v, sa);
            giy += dwp * sample_diy(v, sa);
        }
        const float t3x = T3[((long)n * 2) * hw + pp], t3y = T3[((long)n * 2 + 1) * hw + pp];
        l[2] += fabsf(gcx - t3x) + fabsf(gcy - t3y);
        const float dgx = gix * mx + wn.z * sgn(gcx - t3x), dgy = giy * my + wn.z * sgn(gcy - t3y);
        *reinterpret_cast<float4*>(d_out7 + i * 8) = make_float4(dgx, dgy, dalpha, dcol[0]);
        *reinterpret_cast<float4*>(d_out7 + i * 8 + 4) = make_float4(dcol[1], dcol[2], dcol[3], 0.0f);
    }
#pragma unroll
    for (int k = 0; k < 4; ++k)
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) l[k] += __shfl_xor_sync(0xffffffffu, l[k], off);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) for (int k = 0; k < 4; ++k) red[warp][k] = l[k];
    __syncthreads();
    if (threadIdx.x < 4) {
        double s = 0.0;
        for (int w = 0; w < 8; ++w) s += (double)red[w][threadIdx.x];
        atomicAdd(loss_acc + threadIdx.x, s);
    }
}

// Face student: out4 [P][4] (NHWC) vs target / mask NCHW [N,4,R,R].  loss_acc[0] = sum |o - t|, loss_acc[1] = sum |(t - o) m|
// (l1_loss.py:9-24 L1Loss, :40-58 MaskedL1Loss); d_out = wn.x sgn(o - t) + wn.y sgn((o - t) m) m.
__global__ void __launch_bounds__(256) face_tail_kernel(const float* __restrict__ out4, const float* __restrict__ target,
                                                        const float* __restrict__ mask, int R, int N, float2 wn,
                                                        float* __restrict__ d_out, double* __restrict__ loss_acc) {
    __shared__ float red[8][2];
    const long hw = (long)R * R, total = (long)N * hw;
    float l0 = 0.0f, l1 = 0.0f;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const long pp = i % hw; const int n = (int)(i / hw);
        const float4 o = *reinterpret_cast<const float4*>(out4 + i * 4);
        const float ov[4] = {o.x, o.y, o.z, o.w};
        float g[4];
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            const long ti = ((long)n * 4 + c) * hw + pp;
            const float d = ov[c] - target[ti], m = mask[ti];
            l0 += fabsf(d); l1 += fabsf(d * m);
            g[c] = wn.x * sgn(d) + wn.y * sgn(d * m) * m;
        }
        *reinterpret_cast<float4*>(d_out + i * 4) = make_float4(g[0], g[1], g[2], g[3]);
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) { l0 += __shfl_xor_sync(0xffffffffu, l0, off); l1 += __shfl_xor_sync(0xffffffffu, l1, off); }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) { red[warp][0] = l0; red[warp][1] = l1; }
    __syncthreads();
    if (threadIdx.x < 2) {
        double s = 0.0;
        for (int w = 0; w < 8; ++w) s += (double)red[w][threadIdx.x];
        atomicAdd(loss_acc + threadIdx.x, s);
    }
}

// Tail of the backward from arbitrary upstream gradients (module-level autograd): recomputes the sample of
// train_tail_kernel and applies the chain rule of blended = (1 - alpha) warped + alpha colour (alpha and colour raw,
// siren_morpher_03.py:127-131).  g_bl / g_wp / g_col [N,4,R,R], g_al [N,1,R,R], g_grid [N,2,R,R] (NCHW; NULL = zero).
// d_out7: [P][8] in the layout of out7.
__global__ void __launch_bounds__(256) grad_tail_kernel(const float* __restrict__ out7, ImgView image, const float* __restrict__ g_bl,
                                                        const float* __restrict__ g_al, const float* __restrict__ g_col,
                                                        const float* __restrict__ g_wp, const float* __restrict__ g_grid,
                                                        const float* __restrict__ base, int R, float* __restrict__ d_out7) {
    const long hw = (long)R * R, total = image.N * hw;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int x = (int)(i % R), y = (int)((i / R) % R), n = (int)(i / hw);
        const long pp = (long)y * R + x;
        const float4 oa = *reinterpret_cast<const float4*>(out7 + i * 8), ob = *reinterpret_cast<const float4*>(out7 + i * 8 + 4);
        const float gcx = oa.x, gcy = oa.y, alpha = oa.z;
        const float col[4] = {oa.w, ob.x, ob.y, ob.z};
        const SampleAt sa = sample_locate(base, x, y, gcx, gcy, R);
        float gix = 0.0f, giy = 0.0f, dalpha = g_al ? g_al[(long)n * hw + pp] : 0.0f, dcol[4];
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            const long ti = ((long)n * 4 + c) * hw + pp;
            const Corners v = sample_corners(image.p + n * image.sn + c * image.sc, image.sh, sa);
            const float wp = sample_value(v, sa);
            const float gbl = g_bl ? g_bl[ti] : 0.0f;
            const float dwp = gbl * (1.0f - alpha) + (g_wp ? g_wp[ti] : 0.0f);
            dalpha += gbl * (col[c] - wp);
            dcol[c] = gbl * alpha + (g_col ? g_col[ti] : 0.0f);
            gix += dwp * sample_dix(v, sa);
            giy += dwp * sample_diy(v, sa);
        }
        float dgx = gix * sa.mx, dgy = giy * sa.my;
        if (g_grid) { dgx += g_grid[((long)n * 2) * hw + pp]; dgy += g_grid[((long)n * 2 + 1) * hw + pp]; }
        *reinterpret_cast<float4*>(d_out7 + i * 8) = make_float4(dgx, dgy, dalpha, dcol[0]);
        *reinterpret_cast<float4*>(d_out7 + i * 8 + 4) = make_float4(dcol[1], dcol[2], dcol[3], 0.0f);
    }
}

// d_out [P][4] (NHWC, what the face backward reads) from the upstream gradient g [N,4,R,R] (NCHW)
__global__ void __launch_bounds__(256) face_grad_layout_kernel(const float* __restrict__ g, int R, int N, float* __restrict__ d_out) {
    const long hw = (long)R * R, total = (long)N * hw;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const long pp = i % hw, n = i / hw;
        const float* gi = g + n * 4 * hw + pp;
        *reinterpret_cast<float4*>(d_out + i * 4) = make_float4(gi[0], gi[hw], gi[2 * hw], gi[3 * hw]);
    }
}

// ---------------------------------------------------------------------------------------------- input gradients
// d(image) of warped = grid_sample(image, base + grid_change) (bilinear, border, align_corners=False) through blended =
// (1 - alpha) warped + alpha colour: each output pixel scatters its bilinear weights x (g_bl (1 - alpha) + g_wp) into the
// corners it sampled.  grid_change [N,2,R,R] and alpha [N,1,R,R] are the values the forward returned, and the corners and
// weights are located with the inference tail's arithmetic (gs_locate / gs_sample), so d(image) is the exact adjoint of the
// returned warp.  Out-of-range corners are skipped, as the forward skips them.  g_bl / g_wp [N,4,R,R] NCHW, NULL = zero.
// d_nhwc: [N][R][R][4], zeroed by the caller; one red.global.add.v4.f32 per corner.  The float atomics make the result
// not bit-reproducible run to run (like torch's CUDA grid_sample backward).  Measured against 16 scalar reds per pixel
// straight into NCHW (H100 80GB HBM3, 700 W; zeroing and layout pass included, one 512x512 sample): 20.5 vs 24.3 us for a
// gently varying grid, 22.7 vs 51.9 us for a rough one; the scalar form is faster only on the identity grid (13.5 vs 16.6).
__global__ void __launch_bounds__(256) image_grad_kernel(const float* __restrict__ grid_change, const float* __restrict__ alpha,
                                                         const float* __restrict__ g_bl, const float* __restrict__ g_wp,
                                                         const float* __restrict__ base, int R, int N, float* __restrict__ d_nhwc) {
    const long hw = (long)R * R, total = (long)N * hw;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int x = (int)(i % R), y = (int)((i / R) % R), n = (int)(i / hw);
        const long pp = i - (long)n * hw;
        const GsTap t = gs_locate(base[x], base[y], grid_change[(2L * n) * hw + pp], grid_change[(2L * n + 1) * hw + pp], R, R);
        const float om = g_bl ? 1.0f - alpha[i] : 0.0f;
        float dw[4];
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            const long ti = ((long)n * 4 + c) * hw + pp;
            dw[c] = (g_bl ? g_bl[ti] * om : 0.0f) + (g_wp ? g_wp[ti] : 0.0f);
        }
        const float wx1 = __fsub_rn(t.ix, t.fx), wx0 = __fsub_rn(__fadd_rn(t.fx, 1.0f), t.ix);
        const float wy1 = __fsub_rn(t.iy, t.fy), wy0 = __fsub_rn(__fadd_rn(t.fy, 1.0f), t.iy);
        const float wnw = __fmul_rn(wx0, wy0), wne = __fmul_rn(wx1, wy0), wsw = __fmul_rn(wx0, wy1), wse = __fmul_rn(wx1, wy1);
        const bool xin = (t.x0 + 1) < R, yin = (t.y0 + 1) < R;
        float4* d = reinterpret_cast<float4*>(d_nhwc) + n * hw + (long)t.y0 * R + t.x0;
        atomicAdd(d, make_float4(wnw * dw[0], wnw * dw[1], wnw * dw[2], wnw * dw[3]));
        if (xin) atomicAdd(d + 1, make_float4(wne * dw[0], wne * dw[1], wne * dw[2], wne * dw[3]));
        if (yin) atomicAdd(d + R, make_float4(wsw * dw[0], wsw * dw[1], wsw * dw[2], wsw * dw[3]));
        if (xin && yin) atomicAdd(d + R + 1, make_float4(wse * dw[0], wse * dw[1], wse * dw[2], wse * dw[3]));
    }
}

// [N][hw][4] (NHWC) -> [N][4][hw] (NCHW)
__global__ void __launch_bounds__(256) nhwc4_to_nchw_kernel(const float* __restrict__ src, long hw, int N, float* __restrict__ dst) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < (long)N * hw; i += (long)gridDim.x * blockDim.x) {
        const long n = i / hw, pp = i - n * hw;
        const float4 v = reinterpret_cast<const float4*>(src)[i];
        float* o = dst + n * 4 * hw + pp;
        o[0] = v.x; o[hw] = v.y; o[2 * hw] = v.z; o[3 * hw] = v.w;
    }
}

// d(pose), stage 1: the pose enters only as columns col0 .. col0 + npose - 1 of each level's first layer, so
// d pose[n][k] = sum_levels sum_c S[n][c] W0[c][col0 + k] with S[n][c] = sum over sample n's pixels of the first layer's dz.
// This stage sums dz [N][hw][C] over chunks of POSE_CHUNK pixels in a fixed order: part[n][chunk][C] (fp32).  Grid
// (hw / POSE_CHUNK, N).  C % 4 == 0, C <= 1024.  No atomics: d(pose) is bit-reproducible and independent of the batch.
constexpr int POSE_CHUNK = 256;
__global__ void __launch_bounds__(256) pose_colsum_kernel(const float* __restrict__ dz, int C, long hw, float* __restrict__ part) {
    __shared__ float4 red[256];
    const int cq = C >> 2, PL = 256 / cq;
    const int tid = threadIdx.x, pl = tid / cq, q = tid - pl * cq;
    const long n = blockIdx.y, chunk = blockIdx.x;
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    if (pl < PL) {
        const float* src = dz + (n * hw + chunk * POSE_CHUNK) * C + 4 * q;
        for (int r = pl; r < POSE_CHUNK; r += PL) {
            const float4 v = *reinterpret_cast<const float4*>(src + (long)r * C);
            s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
        }
    }
    red[tid] = s;
    __syncthreads();
    if (pl == 0) {
        float4 acc = red[q];
        for (int j = 1; j < PL; ++j) {
            const float4 v = red[j * cq + q];
            acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
        }
        *reinterpret_cast<float4*>(part + (n * gridDim.x + chunk) * C + 4 * q) = acc;
    }
}

// d(pose), stage 2: one block per sample.  S[l][c] = the chunk partials of level l summed in fp64 (fixed order), then
// d pose[n][k] = sum_l sum_c S[l][c] W_l[c][col0_l + k] in fp64 with the fp32 weights of the flat parameter buffer.
struct PoseLevel {
    const float* part;     // [N][nchunk][C] from pose_colsum_kernel
    const float* W;        // first-layer weight [nreal][kreal]
    int nchunk, C, nreal, kreal, col0;
};
struct PoseGrad {
    PoseLevel lv[3];
    int nl = 0, npose = 0;
};
constexpr int POSE_PROJECT_THREADS = 384;
__global__ void __launch_bounds__(POSE_PROJECT_THREADS) pose_project_kernel(const PoseGrad p, float* __restrict__ dpose) {
    __shared__ double S[3][POSE_PROJECT_THREADS];
    const int n = blockIdx.x, tid = threadIdx.x;
#pragma unroll
    for (int l = 0; l < 3; ++l) {
        if (l >= p.nl) break;
        const PoseLevel& L = p.lv[l];
        if (tid < L.nreal) {
            const float* src = L.part + (long)n * L.nchunk * L.C + tid;
            double s = 0.0;
            for (int k = 0; k < L.nchunk; ++k) s += (double)src[(long)k * L.C];
            S[l][tid] = s;
        }
    }
    __syncthreads();
    if (tid < p.npose) {
        double acc = 0.0;
#pragma unroll
        for (int l = 0; l < 3; ++l) {
            if (l >= p.nl) break;
            const PoseLevel& L = p.lv[l];
            for (int c = 0; c < L.nreal; ++c) acc += S[l][c] * (double)L.W[(long)c * L.kreal + L.col0 + tid];
        }
        dpose[(long)n * p.npose + tid] = (float)acc;
    }
}

// torch.optim.Adam (no weight decay, no amsgrad): optimizer_factories.py:9-17 (betas 0.9 / 0.999, eps 1e-8)
__global__ void adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v, long n,
                            float lr, float b1, float b2, float eps, float bc1, float bc2, float gscale) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
        const float gi = g[i] * gscale;
        const float mi = b1 * m[i] + (1.0f - b1) * gi;
        const float vi = b2 * v[i] + (1.0f - b2) * gi * gi;
        m[i] = mi; v[i] = vi;
        const float denom = sqrtf(vi) / sqrtf(bc2) + eps;
        p[i] -= (lr / bc1) * (mi / denom);
    }
}

inline int grid_for(long total, int cap = 148 * 8) { return (int)std::max<long>(1, std::min<long>((total + 255) / 256, cap)); }

struct Dense {             // one 1x1 layer of the student in the flat parameter buffer
    long w_off, b_off;     // offsets (floats)
    int nreal, kreal;      // reference [Cout][Cin]
    int npad, kpad;        // channel counts of the activation tensors (multiples of 4)
};

View mk(Pool* pool, int N, int R, int C) {
    View v; v.N = N; v.H = R; v.W = R; v.C = C; v.ld = C; v.p = pool->alloc((size_t)N * R * R * C);
    return v;
}

// y = x * W^T (+ bias): 1x1 conv through the shared conv dispatcher (wgmma when available)
void dense_gemm(Runtime& rt, const float* W, int nreal, int kreal, bool transpose, const float* bias_padded,
                const View& x, const View& y) {
    ConvWeights cw;
    conv_describe(cw, CONV_1x1, x.C, y.C);
    cw.w = rt.scratch->alloc(conv_packed_floats(cw));
    cw.tf32_rounded = true;
    cw.dynamic = true;
    pack_dense_kernel<<<64, 256, 0, rt.stream>>>(W, nreal, kreal, transpose ? 1 : 0, cw.w, cw.cout_pad, cw.cin_pad);
    THA4_LAUNCH_CHECK();
    cw.bias = const_cast<float*>(bias_padded);
    ConvArgs a;
    a.in = x; a.out = y; a.strict = 0;
    const size_t ws = conv_workspace_floats(cw, a);
    if (ws) { a.ws = rt.scratch->alloc(ws); a.ws_floats = ws; }
    conv_forward(cw, a, rt.stream);
}

// weight and bias gradients of layer d: dW += dz^T x, db += column sums of dz
void dense_wgrad(cudaStream_t s, const View& dz, const View& x, const Dense& d, float* grads) {
    const long Pn = (long)dz.N * dz.H * dz.W;
    const int psplit = (int)std::max<long>(1, std::min<long>(64, Pn / 4096));
    dim3 grid(ceil_div(dz.C, 64), ceil_div(x.C, 64), psplit);
    wgrad_kernel<<<grid, 128, 0, s>>>(dz.p, dz.C, x.p, x.C, Pn, d.nreal, d.kreal, grads + d.w_off);
    THA4_LAUNCH_CHECK();
    colsum_kernel<<<std::min<long>(148, std::max<long>(1, Pn / 512)), 256, 0, s>>>(dz.p, Pn, dz.C, d.nreal, grads + d.b_off);
    THA4_LAUNCH_CHECK();
}

// d(pose) stage 1 for one level: chunk sums of the first layer's dz (layer d; the pose columns start at col0)
void pose_colsum(Runtime& rt, const View& dz, const Dense& d, const float* params, int col0, PoseGrad& pg) {
    const long hw = (long)dz.H * dz.W;
    THA4_REQUIRE(hw % POSE_CHUNK == 0 && dz.C % 4 == 0 && dz.C <= 1024 && d.nreal <= POSE_PROJECT_THREADS, "pose gradient: level shape");
    PoseLevel& L = pg.lv[pg.nl++];
    L.nchunk = (int)(hw / POSE_CHUNK); L.C = dz.C; L.nreal = d.nreal; L.kreal = d.kreal; L.col0 = col0;
    L.W = params + d.w_off;
    float* part = rt.persist->alloc((size_t)dz.N * L.nchunk * L.C);
    L.part = part;
    pose_colsum_kernel<<<dim3(L.nchunk, dz.N), 256, 0, rt.stream>>>(dz.p, dz.C, hw, part);
    THA4_LAUNCH_CHECK();
}

// d(pose) stage 2: dpose [N][npose], overwritten
void pose_project(cudaStream_t s, const PoseGrad& pg, int N, float* dpose) {
    pose_project_kernel<<<N, POSE_PROJECT_THREADS, 0, s>>>(pg, dpose);
    THA4_LAUNCH_CHECK();
}

}  // namespace

// reference layer table of SirenMorpher03 (mode_14.py:108-131), in state_dict order
static void body_layers(Dense (&L)[10]) {
    const int dims[10][2] = {{360, 47}, {360, 360}, {180, 360}, {180, 227}, {180, 180}, {90, 180}, {90, 137}, {90, 90}, {90, 90}, {7, 90}};
    const int npad[10] = {360, 360, 180, 180, 180, 92, 92, 92, 92, 8};
    const int kpad[10] = {48, 360, 360, 228, 180, 180, 140, 92, 92, 92};
    long off = 0;
    for (int i = 0; i < 10; ++i) {
        L[i].nreal = dims[i][0]; L[i].kreal = dims[i][1]; L[i].npad = npad[i]; L[i].kpad = kpad[i];
        L[i].w_off = off; off += (long)dims[i][0] * dims[i][1];
        L[i].b_off = off; off += dims[i][0];
    }
}

long siren_body_param_count() { Dense L[10]; body_layers(L); return L[9].b_off + 7; }

namespace {

constexpr int BODY_RS[3] = {128, 256, 512};
constexpr int BODY_CPREV[3] = {0, 180, 90};     // real channels carried up from the previous level

struct BodyActs {          // what the body backward reads: level inputs, pre-activations z, activations a, head output
    View xin[3], z[3][3], a[3][3], out7;
};

// forward of N images with stored activations (TF32 products)
void body_forward_store(Runtime& rt, const Dense (&L)[10], const float* pose, int pose_ld, int N, const float* params, BodyActs& A) {
    cudaStream_t s = rt.stream;
    Pool* P = rt.persist;
    float* bias_pad[10];
    for (int i = 0; i < 10; ++i) {
        bias_pad[i] = P->alloc(L[i].npad);
        pad_bias_kernel<<<ceil_div(L[i].npad, 128), 128, 0, s>>>(params + L[i].b_off, L[i].nreal, L[i].npad, bias_pad[i]);
        THA4_LAUNCH_CHECK();
    }
    for (int l = 0; l < 3; ++l) {
        const int R = BODY_RS[l];
        A.xin[l] = mk(P, N, R, L[3 * l].kpad);
        const View* prev = l > 0 ? &A.a[l - 1][2] : nullptr;
        level_input_kernel<<<grid_for((long)N * R * R * A.xin[l].C), 256, 0, s>>>(prev ? prev->p : nullptr, BODY_CPREV[l], prev ? prev->ld : 0,
                                                                                pose, pose_ld, base_grid_table(R), R, N, A.xin[l].C, 45,
                                                                                A.xin[l].p);
        THA4_LAUNCH_CHECK();
        for (int j = 0; j < 3; ++j) {
            const Dense& d = L[3 * l + j];
            rt.scratch->reset();
            A.z[l][j] = mk(P, N, R, d.npad);
            A.a[l][j] = mk(P, N, R, d.npad);
            dense_gemm(rt, params + d.w_off, d.nreal, d.kreal, false, bias_pad[3 * l + j], j == 0 ? A.xin[l] : A.a[l][j - 1], A.z[l][j]);
            const long n4 = (long)N * R * R * d.npad / 4;
            sine_forward_kernel<<<grid_for(n4), 256, 0, s>>>(A.z[l][j].p, A.a[l][j].p, n4);
            THA4_LAUNCH_CHECK();
        }
    }
    rt.scratch->reset();
    A.out7 = mk(P, N, 512, 8);
    dense_gemm(rt, params + L[9].w_off, 7, 90, false, bias_pad[9], A.a[2][2], A.out7);
}

// backward from d(out7) [P][8]; accumulates into grads, which the caller zeroes.  grads == NULL: no weight gradients.
// pose_grad != NULL: also the stage-1 chunk sums of d(pose) (the caller runs pose_project).
void body_backward(Runtime& rt, const Dense (&L)[10], const BodyActs& A, const View& d_out, const float* params, float* grads,
                   PoseGrad* pose_grad = nullptr) {
    cudaStream_t s = rt.stream;
    Pool* P = rt.persist;
    const int N = d_out.N;
    // head: out7 = a22 W9^T + b9
    if (grads) dense_wgrad(s, d_out, A.a[2][2], L[9], grads);
    View da = mk(P, N, 512, L[8].npad);
    rt.scratch->reset();
    dense_gemm(rt, params + L[9].w_off, 7, 90, true, nullptr, d_out, da);     // d a22 = d_out W9
    for (int l = 2; l >= 0; --l) {
        const int R = BODY_RS[l];
        for (int j = 2; j >= 0; --j) {
            const Dense& d = L[3 * l + j];
            const long n4 = (long)N * R * R * d.npad / 4;
            sine_backward_kernel<<<grid_for(n4), 256, 0, s>>>(A.z[l][j].p, da.p, n4);       // da -> dz (in place)
            THA4_LAUNCH_CHECK();
            const View& x = (j == 0) ? A.xin[l] : A.a[l][j - 1];
            if (grads) dense_wgrad(s, da, x, d, grads);
            if (j == 0 && pose_grad) pose_colsum(rt, da, d, params, BODY_CPREV[l] + 2, *pose_grad);
            if (j == 0 && l == 0) break;
            View dx = mk(P, N, R, d.kpad);
            rt.scratch->reset();
            dense_gemm(rt, params + d.w_off, d.nreal, d.kreal, true, nullptr, da, dx);   // dx = dz W
            if (j > 0) { da = dx; continue; }
            // level boundary: the first Cprev channels of dx are the gradient of the upsampled previous level
            View dprev = mk(P, N, R / 2, L[3 * l - 1].npad);
            THA4_CUDA_CHECK(cudaMemsetAsync(dprev.p, 0, dprev.pixels() * dprev.C * sizeof(float), s));
            upsample_backward_kernel<<<grid_for((long)N * (R / 2) * (R / 2) * BODY_CPREV[l]), 256, 0, s>>>(dx.p, dx.ld, BODY_CPREV[l], R, N,
                                                                                                        dprev.p, dprev.ld);
            THA4_LAUNCH_CHECK();
            da = dprev;
        }
    }
}

}  // namespace

void siren_body_train_step(Runtime& rt, const ImgView& image, const float* pose, int pose_ld, const float* T0, const float* T2,
                           const float* T3, const float loss_w[4], const float* params, float* grads, double* loss_acc) {
    THA4_REQUIRE(image.H == 512 && image.W == 512 && image.C == 4, "distill: image size");
    cudaStream_t s = rt.stream;
    const int N = image.N;
    Dense L[10];
    body_layers(L);
    const long nparams = L[9].b_off + 7;
    THA4_CUDA_CHECK(cudaMemsetAsync(grads, 0, nparams * sizeof(float), s));
    THA4_CUDA_CHECK(cudaMemsetAsync(loss_acc, 0, 4 * sizeof(double), s));
    ProfScope prof(PROF_SIREN, s);
    BodyActs A;
    body_forward_store(rt, L, pose, pose_ld, N, params, A);
    // losses + d(out7)
    View d_out = mk(rt.persist, N, 512, 8);
    const double nb = (double)N * 4 * 512 * 512, ng = (double)N * 2 * 512 * 512;
    const float4 wn = make_float4((float)(loss_w[0] / nb), (float)(loss_w[1] / nb), (float)(loss_w[2] / ng), (float)(loss_w[3] / nb));
    train_tail_kernel<<<grid_for((long)N * 512 * 512), 256, 0, s>>>(A.out7.p, image, T0, T2, T3, base_grid_table(512), 512, wn, d_out.p, loss_acc);
    THA4_LAUNCH_CHECK();
    body_backward(rt, L, A, d_out, params, grads);
}

void siren_body_backward(Runtime& rt, const ImgView& image, const float* pose, int pose_ld, const float* const g[5], const float* params,
                         float* grads, float* d_pose) {
    THA4_REQUIRE(image.H == 512 && image.W == 512 && image.C == 4, "student backward: image size");
    THA4_REQUIRE(image.N >= 1 && image.N <= SIREN_BODY_MAX_BATCH, "student backward: micro-batch must be 1..8");
    cudaStream_t s = rt.stream;
    const int N = image.N;
    Dense L[10];
    body_layers(L);
    ProfScope prof(PROF_SIREN, s);
    BodyActs A;
    body_forward_store(rt, L, pose, pose_ld, N, params, A);
    View d_out = mk(rt.persist, N, 512, 8);
    grad_tail_kernel<<<grid_for((long)N * 512 * 512), 256, 0, s>>>(A.out7.p, image, g[0], g[1], g[2], g[3], g[4], base_grid_table(512), 512,
                                                                   d_out.p);
    THA4_LAUNCH_CHECK();
    PoseGrad pg;
    pg.npose = 45;
    body_backward(rt, L, A, d_out, params, grads, d_pose ? &pg : nullptr);
    if (d_pose) pose_project(s, pg, N, d_pose);
}

void siren_body_image_grad(Runtime& rt, const float* grid_change, const float* alpha, const float* g_bl, const float* g_wp, int N,
                           float* d_image) {
    THA4_REQUIRE(N >= 1 && N <= SIREN_BODY_MAX_BATCH, "student image gradient: micro-batch must be 1..8");
    cudaStream_t s = rt.stream;
    constexpr int R = 512;
    const long hw = (long)R * R;
    if (!g_bl && !g_wp) {               // warped reaches no output that has a gradient
        THA4_CUDA_CHECK(cudaMemsetAsync(d_image, 0, (size_t)N * 4 * hw * sizeof(float), s));
        return;
    }
    float* acc = rt.persist->alloc((size_t)N * hw * 4);
    THA4_CUDA_CHECK(cudaMemsetAsync(acc, 0, (size_t)N * hw * 4 * sizeof(float), s));
    image_grad_kernel<<<grid_for(N * hw), 256, 0, s>>>(grid_change, alpha, g_bl, g_wp, base_grid_table(R), R, N, acc);
    THA4_LAUNCH_CHECK();
    nhwc4_to_nchw_kernel<<<grid_for(N * hw), 256, 0, s>>>(acc, hw, N, d_image);
    THA4_LAUNCH_CHECK();
}

// reference layer table of SirenFaceMorpher00 (mode_14.py:93-105; vanilla/siren.py:60-91), in state_dict order
static void face_layers(Dense (&L)[9]) {
    long off = 0;
    for (int i = 0; i < 9; ++i) {
        L[i].nreal = i == 8 ? 4 : 128; L[i].kreal = i == 0 ? 41 : 128;
        L[i].npad = L[i].nreal; L[i].kpad = i == 0 ? 44 : 128;
        L[i].w_off = off; off += (long)L[i].nreal * L[i].kreal;
        L[i].b_off = off; off += L[i].nreal;
    }
}

long siren_face_param_count() { Dense L[9]; face_layers(L); return L[8].b_off + 4; }

namespace {

constexpr int FACE_R = 128;

struct FaceActs { View xin, z[8], a[8], out4; };

void face_forward_store(Runtime& rt, const Dense (&L)[9], const float* pose, int pose_ld, int N, const float* params, FaceActs& A) {
    cudaStream_t s = rt.stream;
    Pool* P = rt.persist;
    constexpr int R = FACE_R;
    float* bias_pad[9];
    for (int i = 0; i < 9; ++i) {
        bias_pad[i] = P->alloc(L[i].npad);
        pad_bias_kernel<<<1, 128, 0, s>>>(params + L[i].b_off, L[i].nreal, L[i].npad, bias_pad[i]);
        THA4_LAUNCH_CHECK();
    }
    A.xin = mk(P, N, R, L[0].kpad);
    level_input_kernel<<<grid_for((long)N * R * R * A.xin.C), 256, 0, s>>>(nullptr, 0, 0, pose, pose_ld, base_grid_table(R), R, N, A.xin.C, 39,
                                                                          A.xin.p);
    THA4_LAUNCH_CHECK();
    const long n4 = (long)N * R * R * 128 / 4;
    for (int j = 0; j < 8; ++j) {
        rt.scratch->reset();
        A.z[j] = mk(P, N, R, 128);
        A.a[j] = mk(P, N, R, 128);
        dense_gemm(rt, params + L[j].w_off, L[j].nreal, L[j].kreal, false, bias_pad[j], j == 0 ? A.xin : A.a[j - 1], A.z[j]);
        sine_forward_kernel<<<grid_for(n4), 256, 0, s>>>(A.z[j].p, A.a[j].p, n4);
        THA4_LAUNCH_CHECK();
    }
    rt.scratch->reset();
    A.out4 = mk(P, N, R, 4);
    dense_gemm(rt, params + L[8].w_off, 4, 128, false, bias_pad[8], A.a[7], A.out4);
}

// backward from d(out4) [P][4]; accumulates into grads, which the caller zeroes.  grads == NULL: no weight gradients.
// pose_grad != NULL: also the stage-1 chunk sums of d(pose) (the caller runs pose_project).
void face_backward(Runtime& rt, const Dense (&L)[9], const FaceActs& A, const View& d_out, const float* params, float* grads,
                   PoseGrad* pose_grad = nullptr) {
    cudaStream_t s = rt.stream;
    Pool* P = rt.persist;
    constexpr int R = FACE_R;
    const int N = d_out.N;
    const long n4 = (long)N * R * R * 128 / 4;
    if (grads) dense_wgrad(s, d_out, A.a[7], L[8], grads);
    View da = mk(P, N, R, 128);
    rt.scratch->reset();
    dense_gemm(rt, params + L[8].w_off, 4, 128, true, nullptr, d_out, da);       // d a7 = d_out W8
    for (int j = 7; j >= 0; --j) {
        sine_backward_kernel<<<grid_for(n4), 256, 0, s>>>(A.z[j].p, da.p, n4);       // da -> dz (in place)
        THA4_LAUNCH_CHECK();
        if (grads) dense_wgrad(s, da, j == 0 ? A.xin : A.a[j - 1], L[j], grads);
        if (j == 0 && pose_grad) pose_colsum(rt, da, L[0], params, 2, *pose_grad);
        if (j == 0) break;
        View dx = mk(P, N, R, 128);
        rt.scratch->reset();
        dense_gemm(rt, params + L[j].w_off, L[j].nreal, L[j].kreal, true, nullptr, da, dx);   // dx = dz W
        da = dx;
    }
}

}  // namespace

// Face-student distillation step (SURVEY.md section 8 a17): SirenFaceMorpher00 forward with stored activations, L1 +
// eye/mouth-masked L1 against the teacher crop, full backward into a flat gradient buffer.
// Reference: siren_face_morpher_protocols_00.py:48-105, siren_face_morpher_00_trainer.py:112-186.
void siren_face_train_step(Runtime& rt, const float* pose, int pose_ld, int N, const float* target, const float* mask,
                           const float loss_w[2], const float* params, float* grads, double* loss_acc) {
    cudaStream_t s = rt.stream;
    constexpr int R = FACE_R;
    Dense L[9];
    face_layers(L);
    const long nparams = L[8].b_off + 4;
    THA4_CUDA_CHECK(cudaMemsetAsync(grads, 0, nparams * sizeof(float), s));
    THA4_CUDA_CHECK(cudaMemsetAsync(loss_acc, 0, 4 * sizeof(double), s));
    ProfScope prof(PROF_SIREN, s);
    FaceActs A;
    face_forward_store(rt, L, pose, pose_ld, N, params, A);
    // losses + d(out4)
    View d_out = mk(rt.persist, N, R, 4);
    const double nel = (double)N * 4 * R * R;
    face_tail_kernel<<<grid_for((long)N * R * R), 256, 0, s>>>(A.out4.p, target, mask, R, N,
                                                              make_float2((float)(loss_w[0] / nel), (float)(loss_w[1] / nel)), d_out.p, loss_acc);
    THA4_LAUNCH_CHECK();
    face_backward(rt, L, A, d_out, params, grads);
}

void siren_face_backward(Runtime& rt, const float* pose, int pose_ld, int N, const float* grad_output, const float* params, float* grads,
                         float* d_pose) {
    THA4_REQUIRE(N >= 1 && N <= SIREN_FACE_MAX_BATCH, "face student backward: micro-batch must be 1..64");
    cudaStream_t s = rt.stream;
    constexpr int R = FACE_R;
    Dense L[9];
    face_layers(L);
    ProfScope prof(PROF_SIREN, s);
    FaceActs A;
    face_forward_store(rt, L, pose, pose_ld, N, params, A);
    View d_out = mk(rt.persist, N, R, 4);
    face_grad_layout_kernel<<<grid_for((long)N * R * R), 256, 0, s>>>(grad_output, R, N, d_out.p);
    THA4_LAUNCH_CHECK();
    PoseGrad pg;
    pg.npose = 39;
    face_backward(rt, L, A, d_out, params, grads, d_pose ? &pg : nullptr);
    if (d_pose) pose_project(s, pg, N, d_pose);
}

void adam_step(float* params, const float* grads, float* m, float* v, long n, float lr, float beta1, float beta2, float eps,
               int step, float grad_scale, cudaStream_t s) {
    const float bc1 = 1.0f - powf(beta1, (float)step), bc2 = 1.0f - powf(beta2, (float)step);
    adam_kernel<<<grid_for(n), 256, 0, s>>>(params, grads, m, v, n, lr, beta1, beta2, eps, bc1, bc2, grad_scale);
    THA4_LAUNCH_CHECK();
}

}  // namespace tha4
