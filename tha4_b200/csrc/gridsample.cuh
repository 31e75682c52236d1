// Device-side restatement of affine_grid + grid_sample(bilinear, border, align_corners=False) and of bilinear
// interpolate(align_corners=False).  The index arithmetic uses explicit round-to-nearest intrinsics (no FMA
// contraction) so that corner indices and lerp weights are bit-identical to oracle/gridsample_ref.c.
// Reference call sites: nn/image_processing_util.py:13-24,33-54; face_morpher_08.py:142-153; mode_07.py:102,114-115.
#pragma once
#include "common.cuh"

namespace tha4 {

// ((g + 1) * size - 1) / 2 clamped to [0, size-1]   (ATen GridSampler.h grid_sampler_unnormalize + clip_coordinates)
__device__ __forceinline__ float gs_src_index(float g, int size) {
    float v = __fdiv_rn(__fsub_rn(__fmul_rn(__fadd_rn(g, 1.0f), (float)size), 1.0f), 2.0f);
    return fminf((float)(size - 1), fmaxf(v, 0.0f));
}

struct GsTap {
    int x0, y0;
    float ix, iy, fx, fy;
};

__device__ __forceinline__ GsTap gs_locate(float base_x, float base_y, float dxv, float dyv, int W, int H) {
    GsTap t;
    t.ix = gs_src_index(__fadd_rn(base_x, dxv), W);
    t.iy = gs_src_index(__fadd_rn(base_y, dyv), H);
    t.fx = floorf(t.ix); t.fy = floorf(t.iy);
    t.x0 = (int)t.fx; t.y0 = (int)t.fy;
    return t;
}

// Samples C planar channels (stride sc) of one image at tap t.  img points at the sample's channel 0.
template <int C>
__device__ __forceinline__ void gs_sample(const float* __restrict__ img, long sc, long sh, int W, int H, const GsTap& t,
                                          float (&out)[C]) {
    const float wx1 = __fsub_rn(t.ix, t.fx), wx0 = __fsub_rn(__fadd_rn(t.fx, 1.0f), t.ix);
    const float wy1 = __fsub_rn(t.iy, t.fy), wy0 = __fsub_rn(__fadd_rn(t.fy, 1.0f), t.iy);
    const float wnw = __fmul_rn(wx0, wy0), wne = __fmul_rn(wx1, wy0), wsw = __fmul_rn(wx0, wy1), wse = __fmul_rn(wx1, wy1);
    const bool xin = (t.x0 + 1) < W, yin = (t.y0 + 1) < H;
    const long o00 = (long)t.y0 * sh + t.x0;
    const long o01 = xin ? o00 + 1 : o00, o10 = yin ? o00 + sh : o00, o11 = o10 + (xin ? 1 : 0);
    // all 4 * C corner loads are requested before the first is consumed (the offsets are clamped, so every address is valid):
    // with the loads inside the conditionals the drain of the fused tails waited for ~8 separate round trips per pixel
    float v00[C], v01[C], v10[C], v11[C];
#pragma unroll
    for (int c = 0; c < C; ++c) {
        const float* p = img + c * sc;
        v00[c] = __ldg(p + o00); v01[c] = __ldg(p + o01); v10[c] = __ldg(p + o10); v11[c] = __ldg(p + o11);
    }
#pragma unroll
    for (int c = 0; c < C; ++c) {
        float acc = __fmul_rn(v00[c], wnw);
        if (xin) acc = __fadd_rn(acc, __fmul_rn(v01[c], wne));
        if (yin) acc = __fadd_rn(acc, __fmul_rn(v10[c], wsw));
        if (xin && yin) acc = __fadd_rn(acc, __fmul_rn(v11[c], wse));
        out[c] = acc;
    }
}

// Same sampling from an INTERLEAVED copy of the RGBA image (NHWC, `ld` floats per pixel, the four channels 16-byte aligned;
// img points at pixel (0, 0) of the sample): one 16-byte load per corner instead of four 4-byte loads from four planes.
// The planar version needs sixteen 64-bit addresses per pixel; under the register cap of the fused tails the compiler reused
// one address register pair and the loads serialised on its release (ncu source page: the long-scoreboard stalls of the
// drain sat on the IADD3s between the LDGs).  Same products, same order of additions: bit-identical results.
// issue: the four corner pixels of tap t (clamped offsets: every address is valid)
__device__ __forceinline__ void gs_issue4_nhwc(const float* __restrict__ img, int ld, int W, int H, const GsTap& t, float4 (&v)[4]) {
    const bool xin = (t.x0 + 1) < W, yin = (t.y0 + 1) < H;
    const int p00 = t.y0 * W + t.x0;
    const int p01 = p00 + (xin ? 1 : 0), p10 = p00 + (yin ? W : 0), p11 = p10 + (xin ? 1 : 0);
    v[0] = __ldg(reinterpret_cast<const float4*>(img + (size_t)((unsigned)p00 * (unsigned)ld)));
    v[1] = __ldg(reinterpret_cast<const float4*>(img + (size_t)((unsigned)p01 * (unsigned)ld)));
    v[2] = __ldg(reinterpret_cast<const float4*>(img + (size_t)((unsigned)p10 * (unsigned)ld)));
    v[3] = __ldg(reinterpret_cast<const float4*>(img + (size_t)((unsigned)p11 * (unsigned)ld)));
}
// combine: the bilinear blend of the loaded corners, in gs_sample's order of operations
__device__ __forceinline__ void gs_combine4(const GsTap& t, int W, int H, const float4 (&v)[4], float (&out)[4]) {
    const float wx1 = __fsub_rn(t.ix, t.fx), wx0 = __fsub_rn(__fadd_rn(t.fx, 1.0f), t.ix);
    const float wy1 = __fsub_rn(t.iy, t.fy), wy0 = __fsub_rn(__fadd_rn(t.fy, 1.0f), t.iy);
    const float wnw = __fmul_rn(wx0, wy0), wne = __fmul_rn(wx1, wy0), wsw = __fmul_rn(wx0, wy1), wse = __fmul_rn(wx1, wy1);
    const bool xin = (t.x0 + 1) < W, yin = (t.y0 + 1) < H;
    const float v00[4] = {v[0].x, v[0].y, v[0].z, v[0].w}, v01[4] = {v[1].x, v[1].y, v[1].z, v[1].w};
    const float v10[4] = {v[2].x, v[2].y, v[2].z, v[2].w}, v11[4] = {v[3].x, v[3].y, v[3].z, v[3].w};
#pragma unroll
    for (int ch = 0; ch < 4; ++ch) {
        float acc = __fmul_rn(v00[ch], wnw);
        if (xin) acc = __fadd_rn(acc, __fmul_rn(v01[ch], wne));
        if (yin) acc = __fadd_rn(acc, __fmul_rn(v10[ch], wsw));
        if (xin && yin) acc = __fadd_rn(acc, __fmul_rn(v11[ch], wse));
        out[ch] = acc;
    }
}
__device__ __forceinline__ void gs_sample4_nhwc(const float* __restrict__ img, int ld, int W, int H, const GsTap& t, float (&out)[4]) {
    float4 v[4];
    gs_issue4_nhwc(img, ld, W, H, t, v);
    gs_combine4(t, W, H, v, out);
}

// Bilinear sample of one pixel at base + grid change (the arithmetic above), with what its backward needs.
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

// interpolate(bilinear, align_corners=False) source coordinate for one axis.
struct LerpTap { int i0, i1; float l0, l1; };
__device__ __forceinline__ LerpTap lerp_locate(int dst, float scale, int in_size) {
    float f = __fsub_rn(__fmul_rn(scale, __fadd_rn((float)dst, 0.5f)), 0.5f);
    if (f < 0.0f) f = 0.0f;
    LerpTap t;
    t.i0 = (int)f;
    t.i1 = t.i0 + ((t.i0 < in_size - 1) ? 1 : 0);
    t.l1 = __fsub_rn(f, (float)t.i0);
    t.l0 = __fsub_rn(1.0f, t.l1);
    return t;
}
__device__ __forceinline__ float lerp2(const float* __restrict__ im, long sh, const LerpTap& ty, const LerpTap& tx) {
    const float a = __ldg(im + ty.i0 * sh + tx.i0), b = __ldg(im + ty.i0 * sh + tx.i1);
    const float c = __ldg(im + ty.i1 * sh + tx.i0), d = __ldg(im + ty.i1 * sh + tx.i1);
    return __fadd_rn(__fmul_rn(ty.l0, __fadd_rn(__fmul_rn(tx.l0, a), __fmul_rn(tx.l1, b))),
                     __fmul_rn(ty.l1, __fadd_rn(__fmul_rn(tx.l0, c), __fmul_rn(tx.l1, d))));
}

}  // namespace tha4
