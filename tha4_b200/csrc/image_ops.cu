// Image glue kernels: NCHW<->NHWC, strided window copies (crop / paste, mode_07.py:74,89-97; mode_14.py:60-78),
// bilinear resize (mode_07.py:102,114-115), standalone grid_sample, the Upscaler02 prologue and the
// eyebrow-cache image comparison (mode_07.py:56-61).  All HBM-bound, coalesced along x.
#include "ops.cuh"
#include "gridsample.cuh"
#include <map>
#include <mutex>
#include <vector>

namespace tha4 {
namespace {

__global__ void nchw_to_nhwc_kernel(ImgView src, float* __restrict__ dst, int ld) {
    const long total = (long)src.N * src.H * src.W;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int x = (int)(i % src.W);
        long r = i / src.W;
        const int y = (int)(r % src.H);
        const int n = (int)(r / src.H);
        const float* sp = src.p + n * src.sn + y * src.sh + x;
        float* dp = dst + i * ld;
        for (int c = 0; c < src.C; ++c) dp[c] = __ldg(sp + c * src.sc);
    }
}

__global__ void nhwc_to_nchw_kernel(const float* __restrict__ src, int N, int H, int W, int C, int ld, float* __restrict__ dst) {
    const long total = (long)N * C * H * W;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int x = (int)(i % W);
        long r = i / W;
        const int y = (int)(r % H); r /= H;
        const int c = (int)(r % C);
        const int n = (int)(r / C);
        dst[i] = src[(((long)n * H + y) * W + x) * ld + c];
    }
}

__global__ void copy_window_kernel(ImgView src, float* __restrict__ dst, long dn, long dc, long dh) {
    const long total = (long)src.N * src.C * src.H * src.W;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int x = (int)(i % src.W);
        long r = i / src.W;
        const int y = (int)(r % src.H); r /= src.H;
        const int c = (int)(r % src.C);
        const int n = (int)(r / src.C);
        dst[n * dn + c * dc + y * dh + x] = __ldg(src.p + n * src.sn + c * src.sc + y * src.sh + x);
    }
}

template <typename T>
__global__ void tile_vector_kernel(const float* __restrict__ vec, int vec_ld, int P, T* __restrict__ dst, int H, int W,
                                   int C, int ld, long total) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int c = (int)(i % C);
        const long pix = i / C;
        const int n = (int)(pix / ((long)H * W));
        dst[pix * ld + c] = (T)((c < P) ? vec[(long)n * vec_ld + c] : 0.0f);
    }
}

__global__ void convert_f16_kernel(const float* __restrict__ src, int src_ld, __half* __restrict__ dst, int dst_ld, int C, long total) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int c = (int)(i % C);
        const long pix = i / C;
        dst[pix * dst_ld + c] = __float2half_rn(src[pix * src_ld + c]);
    }
}

__global__ void convert_f32_kernel(const __half* __restrict__ src, int src_ld, float* __restrict__ dst, int dst_ld, int C, long total) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int c = (int)(i % C);
        const long pix = i / C;
        dst[pix * dst_ld + c] = __half2float(src[pix * src_ld + c]);
    }
}

// ---- image I/O on either side of the poser (SURVEY 8f-1) ----
// Poser output [B,4,H,W] fp32 in [-1,1] (linear RGB, alpha) -> HWC uint8 sRGB, what the puppeteer apps display
// (character_model_ifacialmocap_puppeteer.py:325-349): clip((x+1)/2, 0, 1) -> linear->sRGB on RGB
// (shion/base/image_util.py:30-32) -> optional blend over an opaque background colour (:377-381) -> * 255 -> uint8
// (`.byte()` truncates; round_mode 1 = rint as convert_output_image_from_torch_to_numpy does, tha4/image_util.py:56).
// One thread per pixel: four coalesced planar loads, one 4-byte store.
__device__ __forceinline__ float linear_to_srgb_f(float x) {
    x = fminf(fmaxf(x, 0.0f), 1.0f);
    return x <= 0.003130804953560372f ? x * 12.92f : 1.055f * powf(x, 1.0f / 2.4f) - 0.055f;
}
__device__ __forceinline__ float srgb_to_linear_f(float x) {
    x = fminf(fmaxf(x, 0.0f), 1.0f);
    return x <= 0.04045f ? x / 12.92f : powf((x + 0.055f) / 1.055f, 2.4f);
}
__global__ void frame_to_srgb8_kernel(const float* __restrict__ frame, long plane, long total, int has_bg, float bg_r, float bg_g, float bg_b,
                                      int round_mode, uchar4* __restrict__ out) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const long n = i / plane, pix = i - n * plane;
        const float* f = frame + n * 4 * plane + pix;
        float c[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) c[k] = fminf(fmaxf((f[k * plane] + 1.0f) / 2.0f, 0.0f), 1.0f);
        float r = linear_to_srgb_f(c[0]), g = linear_to_srgb_f(c[1]), b = linear_to_srgb_f(c[2]), a = c[3];
        if (has_bg) {
            r = r * a + (1.0f - a) * bg_r; g = g * a + (1.0f - a) * bg_g; b = b * a + (1.0f - a) * bg_b; a = 1.0f;
        }
        uchar4 o;
        if (round_mode) { o.x = (unsigned char)rintf(r * 255.0f); o.y = (unsigned char)rintf(g * 255.0f); o.z = (unsigned char)rintf(b * 255.0f); o.w = (unsigned char)rintf(a * 255.0f); }
        else { o.x = (unsigned char)(255.0f * r); o.y = (unsigned char)(255.0f * g); o.z = (unsigned char)(255.0f * b); o.w = (unsigned char)(255.0f * a); }
        out[i] = o;
    }
}
// PNG pixels (HWC uint8 RGBA, sRGB) -> poser input [4,H,W] fp32: / 255, sRGB -> linear, premultiply by alpha, * 2 - 1
// (shion/base/image_util.py:127-162 with scale 2, offset -1).
__global__ void rgba8_to_poser_image_kernel(const uchar4* __restrict__ rgba, long plane, float* __restrict__ out) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < plane; i += (long)gridDim.x * blockDim.x) {
        const uchar4 p = rgba[i];
        const float a = (float)p.w / 255.0f;
        const float r = srgb_to_linear_f((float)p.x / 255.0f) * a, g = srgb_to_linear_f((float)p.y / 255.0f) * a, b = srgb_to_linear_f((float)p.z / 255.0f) * a;
        out[i] = r * 2.0f - 1.0f; out[plane + i] = g * 2.0f - 1.0f; out[2 * plane + i] = b * 2.0f - 1.0f; out[3 * plane + i] = a * 2.0f - 1.0f;
    }
}

__global__ void resize_bilinear_kernel(ImgView src, float* __restrict__ dst, int Ho, int Wo) {
    const float sy = (float)src.H / (float)Ho, sx = (float)src.W / (float)Wo;
    const long total = (long)src.N * src.C * Ho * Wo;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int x = (int)(i % Wo);
        long r = i / Wo;
        const int y = (int)(r % Ho); r /= Ho;
        const int c = (int)(r % src.C);
        const int n = (int)(r / src.C);
        const LerpTap ty = lerp_locate(y, sy, src.H), tx = lerp_locate(x, sx, src.W);
        dst[i] = lerp2(src.p + n * src.sn + c * src.sc, src.sh, ty, tx);
    }
}

__global__ void grid_sample_kernel(ImgView img, const float* __restrict__ gc, const float* __restrict__ bx,
                                   const float* __restrict__ by, float* __restrict__ out, int* __restrict__ x0o,
                                   int* __restrict__ y0o, float* __restrict__ txo, float* __restrict__ tyo) {
    const long hw = (long)img.H * img.W;
    const long total = img.N * hw;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int x = (int)(i % img.W);
        const int y = (int)((i / img.W) % img.H);
        const int n = (int)(i / hw);
        const long pp = (long)y * img.W + x;
        const GsTap t = gs_locate(bx[x], by[y], gc[(n * 2L) * hw + pp], gc[(n * 2L + 1) * hw + pp], img.W, img.H);
        if (x0o) x0o[i] = t.x0;
        if (y0o) y0o[i] = t.y0;
        if (txo) txo[i] = __fsub_rn(t.ix, t.fx);
        if (tyo) tyo[i] = __fsub_rn(t.iy, t.fy);
        if (out) {
            for (int c = 0; c < img.C; ++c) {
                float v[1];
                gs_sample<1>(img.p + n * img.sn + c * img.sc, 0, img.sh, img.W, img.H, t, v);
                out[((long)n * img.C + c) * hw + pp] = v[0];
            }
        }
    }
}

// rest: [N,4,S,S] view; half_posed [N,4,S/2,S/2]; half_grid [N,2,S/2,S/2]; dst NHWC [N,S,S,16].
__global__ void __launch_bounds__(256) upscaler_prologue_kernel(ImgView rest, const float* __restrict__ half_posed,
                                                                const float* __restrict__ half_grid,
                                                                const float* __restrict__ base, float* __restrict__ dst,
                                                                int ld, int Sh) {
    const int S = rest.W;
    const float scale = (float)Sh / (float)S;
    const long hw = (long)S * S, hwh = (long)Sh * Sh;
    const long total = rest.N * hw;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int x = (int)(i % S);
        const int y = (int)((i / S) % S);
        const int n = (int)(i / hw);
        const LerpTap ty = lerp_locate(y, scale, Sh), tx = lerp_locate(x, scale, Sh);
        float posed[4], grid[2], warped[4], r[4];
#pragma unroll
        for (int c = 0; c < 4; ++c) posed[c] = lerp2(half_posed + (n * 4L + c) * hwh, Sh, ty, tx);
#pragma unroll
        for (int c = 0; c < 2; ++c) grid[c] = lerp2(half_grid + (n * 2L + c) * hwh, Sh, ty, tx);
        const GsTap t = gs_locate(base[x], base[y], grid[0], grid[1], S, S);
        gs_sample<4>(rest.p + n * rest.sn, rest.sc, rest.sh, S, S, t, warped);
#pragma unroll
        for (int c = 0; c < 4; ++c) r[c] = __ldg(rest.p + n * rest.sn + c * rest.sc + (long)y * rest.sh + x);
        float4* dp = reinterpret_cast<float4*>(dst + i * ld);
        dp[0] = make_float4(r[0], r[1], r[2], r[3]);
        dp[1] = make_float4(posed[0], posed[1], posed[2], posed[3]);
        dp[2] = make_float4(warped[0], warped[1], warped[2], warped[3]);
        dp[3] = make_float4(grid[0], grid[1], 0.0f, 0.0f);
    }
}

// Adjoint of upscaler_prologue_kernel.  One thread per COARSE pixel (X, Y) of sample n, r = S / Sh fine pixels per axis.
// dx0: NHWC [N,S,S,ld] gradient of the prologue's output [rest | posed | warped | grid | 0 0] (channels 14, 15 unread).
//   drest (NHWC [N,S,S,4], null = not wanted): += channels 0-3 at the thread's own r x r fine pixels, and the grid_sample
//     image adjoint of channels 8-11 scattered into the corners each of them sampled (atomics, as the tail backward);
//   d_posed [N,4,Sh,Sh] / d_grid [N,2,Sh,Sh] (NCHW, null = not wanted): the bilinear x2 adjoint as a GATHER over the fine
//     pixels whose taps read (X, Y) (fixed order, no atomics; the identity when r == 1) of channels 4-7, and of channels
//     12-13 plus the grid_sample grid gradient of channels 8-11 (zero where the border clamp is active).
__global__ void __launch_bounds__(256) upscaler_prologue_bwd_kernel(ImgView rest, const float* __restrict__ half_grid,
                                                                    const float* __restrict__ base, const float* __restrict__ dx0,
                                                                    int ld, float* __restrict__ drest, float* __restrict__ d_posed,
                                                                    float* __restrict__ d_grid, int Sh) {
    const int S = rest.W, r = S / Sh;
    const float scale = (float)Sh / (float)S;
    const long hw = (long)S * S, hwh = (long)Sh * Sh;
    const long total = rest.N * hwh;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int X = (int)(i % Sh);
        const int Y = (int)((i / Sh) % Sh);
        const int n = (int)(i / hwh);
        const float* rn = rest.p + n * rest.sn;
        const float* gn = half_grid + n * 2L * hwh;
        const float* dn = dx0 + n * hw * ld;
        // the fine grid at (x, y), as the forward interpolated it
        auto fine_grid = [&](int x, int y, float& gx, float& gy) {
            const LerpTap ty = lerp_locate(y, scale, Sh), tx = lerp_locate(x, scale, Sh);
            gx = lerp2(gn, Sh, ty, tx);
            gy = lerp2(gn + hwh, Sh, ty, tx);
        };
        if (drest) {
            float* dr = drest + n * hw * 4;
            for (int y = r * Y; y < r * Y + r; ++y)
                for (int x = r * X; x < r * X + r; ++x) {
                    const float* d = dn + ((long)y * S + x) * ld;
                    const float4 di = *reinterpret_cast<const float4*>(d);
                    atomicAdd(reinterpret_cast<float4*>(dr + ((long)y * S + x) * 4), di);
                    const float4 dw = *reinterpret_cast<const float4*>(d + 8);
                    const float g[4] = {dw.x, dw.y, dw.z, dw.w};
                    float gx, gy;
                    fine_grid(x, y, gx, gy);
                    gs_scatter4_nhwc(dr, 4, S, S, gs_locate(base[x], base[y], gx, gy, S, S), g);
                }
        }
        if (!d_posed && !d_grid) continue;
        // fine rows / columns whose taps can read coarse row Y / column X: r Y - (r - 1) .. r Y + 2 (r - 1)
        float ap[4] = {0.f, 0.f, 0.f, 0.f}, ag[2] = {0.f, 0.f};
        for (int y = max(r * Y - (r - 1), 0); y <= min(r * Y + 2 * (r - 1), S - 1); ++y) {
            const float wy = lerp_weight(y, scale, Sh, Y);
            if (wy == 0.0f) continue;
            for (int x = max(r * X - (r - 1), 0); x <= min(r * X + 2 * (r - 1), S - 1); ++x) {
                const float wx = lerp_weight(x, scale, Sh, X);
                if (wx == 0.0f) continue;
                const float w = wy * wx;
                const float* d = dn + ((long)y * S + x) * ld;
                if (d_posed)
#pragma unroll
                    for (int c = 0; c < 4; ++c) ap[c] = fmaf(w, d[4 + c], ap[c]);
                if (d_grid) {
                    float gx, gy;
                    fine_grid(x, y, gx, gy);
                    const SampleAt sa = sample_locate(base, x, y, gx, gy, S);
                    float gix = 0.0f, giy = 0.0f;
#pragma unroll
                    for (int c = 0; c < 4; ++c) {
                        const Corners v = sample_corners(rn + c * rest.sc, rest.sh, sa);
                        gix += d[8 + c] * sample_dix(v, sa);
                        giy += d[8 + c] * sample_diy(v, sa);
                    }
                    ag[0] = fmaf(w, d[12] + gix * sa.mx, ag[0]);
                    ag[1] = fmaf(w, d[13] + giy * sa.my, ag[1]);
                }
            }
        }
        const long o = (long)Y * Sh + X;
        if (d_posed)
#pragma unroll
            for (int c = 0; c < 4; ++c) d_posed[(n * 4L + c) * hwh + o] = ap[c];
        if (d_grid) {
            d_grid[n * 2L * hwh + o] = ag[0];
            d_grid[(n * 2L + 1) * hwh + o] = ag[1];
        }
    }
}

__global__ void images_differ_kernel(const float* __restrict__ a, const float* __restrict__ b, size_t n, int* flag) {
    bool d = false;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        d |= fabsf(a[i] - b[i]) > 0.0f;
    if (__syncthreads_or(d) && threadIdx.x == 0) atomicOr(flag, 1);
}

inline int grid_for(long total) { return (int)std::min<long>((total + 255) / 256, 148L * 8); }

}  // namespace

void base_grid_host(int W, float* out) {
    // linspace(-1, 1, W) * (W - 1) / W, scalar formula (see oracle/gridsample_ref.c tha4o_base_grid)
    volatile float step = (1.0f - (-1.0f)) / (float)(W - 1);
    const int half = W / 2;
    for (int i = 0; i < W; ++i) {
        volatile float prod = (i < half) ? step * (float)i : step * (float)(W - 1 - i);
        volatile float v = (i < half) ? (-1.0f + prod) : (1.0f - prod);
        volatile float u = v * (float)(W - 1);
        out[i] = u / (float)W;
    }
}

const float* base_grid_table(int size) {
    static std::mutex mu;
    static std::map<std::pair<int, int>, float*> all_tables;      // (device, size): device pointers are per device
    std::lock_guard<std::mutex> lock(mu);
    const std::pair<int, int> key(current_device(), size);
    auto& tables = all_tables;
    auto it = tables.find(key);
    if (it != tables.end()) return it->second;
    std::vector<float> h(size);
    base_grid_host(size, h.data());
    float* d = nullptr;
    THA4_CUDA_CHECK(cudaMalloc(&d, size * sizeof(float)));
    THA4_CUDA_CHECK(cudaMemcpy(d, h.data(), size * sizeof(float), cudaMemcpyHostToDevice));
    tables[key] = d;
    return d;
}

void nchw_to_nhwc(const ImgView& src, const View& dst, cudaStream_t s) {
    THA4_REQUIRE(dst.C == src.C && dst.H == src.H && dst.W == src.W && dst.N == src.N, "nchw_to_nhwc: dims");
    nchw_to_nhwc_kernel<<<grid_for((long)src.N * src.H * src.W), 256, 0, s>>>(src, dst.p, dst.ld);
    THA4_LAUNCH_CHECK();
}

void nhwc_to_nchw(const View& src, float* dst, cudaStream_t s) {
    nhwc_to_nchw_kernel<<<grid_for((long)src.N * src.C * src.H * src.W), 256, 0, s>>>(src.p, src.N, src.H, src.W, src.C, src.ld, dst);
    THA4_LAUNCH_CHECK();
}

void copy_window(const ImgView& src, float* dst, long dn, long dc, long dh, cudaStream_t s) {
    copy_window_kernel<<<grid_for((long)src.N * src.C * src.H * src.W), 256, 0, s>>>(src, dst, dn, dc, dh);
    THA4_LAUNCH_CHECK();
}

void tile_vector(const float* vec, int vec_ld, int P, const View& dst, cudaStream_t s) {
    const long total = (long)dst.N * dst.H * dst.W * dst.C;
    if (dst.f16) tile_vector_kernel<__half><<<grid_for(total), 256, 0, s>>>(vec, vec_ld, P, dst.hp(), dst.H, dst.W, dst.C, dst.ld, total);
    else tile_vector_kernel<float><<<grid_for(total), 256, 0, s>>>(vec, vec_ld, P, dst.p, dst.H, dst.W, dst.C, dst.ld, total);
    THA4_LAUNCH_CHECK();
}

void convert_f16(const View& src, const View& dst, cudaStream_t s) {
    THA4_REQUIRE(!src.f16 && dst.f16 && src.C == dst.C && src.pixels() == dst.pixels(), "convert_f16: views");
    const long total = (long)src.pixels() * src.C;
    convert_f16_kernel<<<grid_for(total), 256, 0, s>>>(src.p, src.ld, dst.hp(), dst.ld, src.C, total);
    THA4_LAUNCH_CHECK();
}

void convert_flat_f16(const float* src, __half* dst, long n, cudaStream_t s) {
    convert_f16_kernel<<<grid_for(n), 256, 0, s>>>(src, 1, dst, 1, 1, n);
    THA4_LAUNCH_CHECK();
}
void convert_flat_f32(const __half* src, float* dst, long n, cudaStream_t s) {
    convert_f32_kernel<<<grid_for(n), 256, 0, s>>>(src, 1, dst, 1, 1, n);
    THA4_LAUNCH_CHECK();
}
void convert_f32(const View& src, const View& dst, cudaStream_t s) {
    THA4_REQUIRE(src.f16 && !dst.f16 && src.C == dst.C && src.pixels() == dst.pixels(), "convert_f32: views");
    const long total = (long)src.pixels() * src.C;
    convert_f32_kernel<<<grid_for(total), 256, 0, s>>>(src.hp(), src.ld, dst.p, dst.ld, src.C, total);
    THA4_LAUNCH_CHECK();
}

void frame_to_srgb8(const float* frame, int B, int H, int W, int background, int round_mode, unsigned char* out, cudaStream_t s) {
    THA4_REQUIRE(background >= 0 && background <= 4, "background: 0 none, 1 green, 2 blue, 3 black, 4 white");
    const float bg[5][3] = {{0, 0, 0}, {0, 1, 0}, {0, 0, 1}, {0, 0, 0}, {1, 1, 1}};
    const long plane = (long)H * W, total = plane * B;
    frame_to_srgb8_kernel<<<grid_for(total), 256, 0, s>>>(frame, plane, total, background != 0, bg[background][0], bg[background][1], bg[background][2],
                                                        round_mode, reinterpret_cast<uchar4*>(out));
    THA4_LAUNCH_CHECK();
}

void rgba8_to_poser_image(const unsigned char* rgba, int H, int W, float* out, cudaStream_t s) {
    const long plane = (long)H * W;
    rgba8_to_poser_image_kernel<<<grid_for(plane), 256, 0, s>>>(reinterpret_cast<const uchar4*>(rgba), plane, out);
    THA4_LAUNCH_CHECK();
}

void resize_bilinear(const ImgView& src, float* dst, int Ho, int Wo, cudaStream_t s) {
    resize_bilinear_kernel<<<grid_for((long)src.N * src.C * Ho * Wo), 256, 0, s>>>(src, dst, Ho, Wo);
    THA4_LAUNCH_CHECK();
}

void grid_sample(const ImgView& image, const float* grid_change, float* out, int* x0, int* y0, float* tx, float* ty,
                 cudaStream_t s) {
    const float* bx = base_grid_table(image.W);
    const float* by = base_grid_table(image.H);
    grid_sample_kernel<<<grid_for((long)image.N * image.H * image.W), 256, 0, s>>>(image, grid_change, bx, by, out, x0, y0, tx, ty);
    THA4_LAUNCH_CHECK();
}

void upscaler_prologue(const ImgView& rest, const float* half_posed, const float* half_grid, int coarse_size,
                       const View& dst, cudaStream_t s) {
    THA4_REQUIRE(coarse_size == rest.H || coarse_size * 2 == rest.H, "upscaler_prologue: coarse size");
    THA4_REQUIRE(rest.C == 4 && rest.H == rest.W && dst.C == 16 && dst.H == rest.H && dst.ld % 4 == 0, "upscaler_prologue: dims");
    upscaler_prologue_kernel<<<grid_for((long)rest.N * rest.H * rest.W), 256, 0, s>>>(rest, half_posed, half_grid,
                                                                                      base_grid_table(rest.W), dst.p, dst.ld, coarse_size);
    THA4_LAUNCH_CHECK();
}

void upscaler_prologue_backward(const ImgView& rest, const float* half_grid, int coarse_size, const View& dx0, float* drest,
                                float* d_posed, float* d_grid, cudaStream_t s) {
    THA4_REQUIRE(coarse_size == rest.H || coarse_size * 2 == rest.H, "upscaler_prologue_backward: coarse size");
    THA4_REQUIRE(rest.C == 4 && rest.H == rest.W && dx0.C >= 14 && dx0.H == rest.H && dx0.W == rest.W && dx0.N == rest.N &&
                 !dx0.f16 && dx0.ld % 4 == 0, "upscaler_prologue_backward: dims");
    upscaler_prologue_bwd_kernel<<<grid_for((long)rest.N * coarse_size * coarse_size), 256, 0, s>>>(
        rest, half_grid, base_grid_table(rest.W), dx0.p, dx0.ld, drest, d_posed, d_grid, coarse_size);
    THA4_LAUNCH_CHECK();
}

bool images_differ(const float* a, const float* b, size_t n, int* dev_flag, cudaStream_t s) {
    THA4_CUDA_CHECK(cudaMemsetAsync(dev_flag, 0, sizeof(int), s));
    images_differ_kernel<<<grid_for((long)n), 256, 0, s>>>(a, b, n, dev_flag);
    THA4_LAUNCH_CHECK();
    int h = 0;
    THA4_CUDA_CHECK(cudaMemcpyAsync(&h, dev_flag, sizeof(int), cudaMemcpyDeviceToHost, s));
    THA4_CUDA_CHECK(cudaStreamSynchronize(s));
    return h != 0;
}

}  // namespace tha4
