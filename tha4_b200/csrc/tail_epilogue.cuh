// Per-pixel epilogue of the fused decoder tails, shared by the fp32 (mma.sync, strict-capable) and the wgmma kernels:
// head outputs of ONE pixel -> sigmoid / tanh -> affine_grid + grid_sample of the RGBA image -> alpha blends -> planar
// NCHW stores of every tensor the network returns.  Reference: eyebrow_decomposer_00.py:49-64,
// eyebrow_morphing_combiner_00.py:51-72, face_morpher_08.py:170-193, morpher_00.py:53-66, upscaler_02.py:84-96.
#pragma once
#include "ops.cuh"
#include "gridsample.cuh"

namespace tha4 {

__device__ __forceinline__ void store4(float* out, long plane, long pix, const float (&v)[4]) {
#pragma unroll
    for (int c = 0; c < 4; ++c) out[c * plane + pix] = v[c];
}

// o[0 .. TAIL_CO_PAD): head conv outputs (bias added) of pixel (y, x) of sample n, in the channel order of `KIND`.
template <int KIND>
__device__ __forceinline__ void tail_epilogue(const float (&o)[TAIL_CO_PAD], int n, int y, int x, int S, const ImgView& img0, const ImgView& img1,
                                              const float* __restrict__ base, float* o0, float* o1, float* o2, float* o3, float* o4,
                                              float* o5, float* o6, float* o7,
                                              const float* __restrict__ g0 = nullptr, int g0_ld = 0, const float* __restrict__ g1 = nullptr, int g1_ld = 0,
                                              const float4 (*pre)[4] = nullptr) {
    // g0 / g1: optional interleaved (NHWC) copies of img0 / img1 (channel 0 of pixel (0,0) of sample 0; per-sample stride
    // S * S * ld floats): the gathers and the per-pixel image reads then take one 16-byte load each (gs_sample4_nhwc)
    const long plane = (long)S * S, pix = (long)y * S + x;
    // pre: the four corner pixels, already requested by tail_gather_issue (the caller did other work while they travelled)
    auto sample0 = [&](const GsTap& t, float (&w)[4]) {
        if (pre) gs_combine4(t, S, S, *pre, w);
        else if (g0) gs_sample4_nhwc(g0 + (size_t)n * S * S * g0_ld, g0_ld, S, S, t, w);
        else gs_sample<4>(img0.p + n * img0.sn, img0.sc, img0.sh, S, S, t, w);
    };
    float* p0 = o0 + n * 4 * plane;   // most outputs are 4-channel; single/dual-channel ones are offset below
    if (KIND == TAIL_UNET) {
        // o: direct(0..3) grid_change(4,5) alpha-logit(6)
        float direct[4] = {o[0], o[1], o[2], o[3]};
        const float alpha = sigmoid_f(o[6]);
        const GsTap t = gs_locate(base[x], base[y], o[4], o[5], S, S);
        float warped[4], merged[4];
        sample0(t, warped);
#pragma unroll
        for (int c = 0; c < 4; ++c) merged[c] = direct[c] * alpha + warped[c] * (1.0f - alpha);
        store4(p0, plane, pix, merged);
        o1[n * plane + pix] = alpha;
        store4(o2 + n * 4 * plane, plane, pix, warped);
        o3[(n * 2L) * plane + pix] = o[4];
        o3[(n * 2L + 1) * plane + pix] = o[5];
        store4(o4 + n * 4 * plane, plane, pix, direct);
    } else if (KIND == TAIL_DECOMPOSER) {
        // o: bg_alpha(0) bg_color(1..4) eb_alpha(5) eb_color(6..9)
        float img[4], bgc[4], ebc[4], bgl[4], ebl[4];
#pragma unroll
        for (int c = 0; c < 4; ++c) img[c] = __ldg(img0.p + n * img0.sn + c * img0.sc + (long)y * img0.sh + x);
        const float bga = sigmoid_f(o[0]), eba = sigmoid_f(o[5]);
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            bgc[c] = tanhf(o[1 + c]); ebc[c] = tanhf(o[6 + c]);
            bgl[c] = bgc[c] * bga + img[c] * (1.0f - bga);
            ebl[c] = img[c] * eba + ebc[c] * (1.0f - eba);     // apply_color_change(alpha, image, color): roles swapped
        }
        store4(p0, plane, pix, ebl);
        o1[n * plane + pix] = eba;
        store4(o2 + n * 4 * plane, plane, pix, ebc);
        store4(o3 + n * 4 * plane, plane, pix, bgl);
        o4[n * plane + pix] = bga;
        store4(o5 + n * 4 * plane, plane, pix, bgc);
    } else if (KIND == TAIL_COMBINER) {
        // o: grid(0,1) alpha(2) color(3..6) combine_alpha(7); img0 = eyebrow layer (warped), img1 = background layer
        const GsTap t = gs_locate(base[x], base[y], o[0], o[1], S, S);
        float warped[4], color[4], morphed[4], bgv[4], e0[4], e1[4];
        sample0(t, warped);
        const float alpha = sigmoid_f(o[2]), ca = sigmoid_f(o[7]);
        if (g1) {
            const float4 b4 = __ldg(reinterpret_cast<const float4*>(g1 + ((size_t)n * S * S + (size_t)y * S + x) * g1_ld));
            bgv[0] = b4.x; bgv[1] = b4.y; bgv[2] = b4.z; bgv[3] = b4.w;
        } else {
#pragma unroll
            for (int c = 0; c < 4; ++c) bgv[c] = __ldg(img1.p + n * img1.sn + c * img1.sc + (long)y * img1.sh + x);
        }
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            color[c] = tanhf(o[3 + c]);
            morphed[c] = color[c] * alpha + warped[c] * (1.0f - alpha);
        }
        const float a2 = (morphed[3] + 1.0f) / 2.0f;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            e0[c] = morphed[c] * ca + bgv[c] * (1.0f - ca);
            e1[c] = morphed[c] * a2 + bgv[c] * (1.0f - a2);
        }
        e0[3] = bgv[3]; e1[3] = bgv[3];
        store4(p0, plane, pix, e0);
        o1[n * plane + pix] = ca;
        store4(o2 + n * 4 * plane, plane, pix, e1);
        store4(o3 + n * 4 * plane, plane, pix, morphed);
        o4[n * plane + pix] = alpha;
        store4(o5 + n * 4 * plane, plane, pix, color);
        store4(o6 + n * 4 * plane, plane, pix, warped);
        o7[(n * 2L) * plane + pix] = o[0];
        o7[(n * 2L + 1) * plane + pix] = o[1];
    } else {  // TAIL_FACE
        // o: grid(0,1) im_color(2..5) im_alpha(6) eye_color(7..10) eye_alpha(11)
        const GsTap t = gs_locate(base[x], base[y], o[0], o[1], S, S);
        float im0[4], imc[4], im1[4], eyc[4], outv[4];
        sample0(t, im0);
        const float ima = sigmoid_f(o[6]), eya = sigmoid_f(o[11]);
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            imc[c] = tanhf(o[2 + c]); eyc[c] = tanhf(o[7 + c]);
            im1[c] = imc[c] * ima + im0[c] * (1.0f - ima);
            outv[c] = eyc[c] * eya + im1[c] * (1.0f - eya);
        }
        store4(p0, plane, pix, outv);
        o1[n * plane + pix] = eya;
        store4(o2 + n * 4 * plane, plane, pix, eyc);
        store4(o3 + n * 4 * plane, plane, pix, im1);
        o4[n * plane + pix] = ima;
        store4(o5 + n * 4 * plane, plane, pix, imc);
        store4(o6 + n * 4 * plane, plane, pix, im0);
        o7[(n * 2L) * plane + pix] = o[0];
        o7[(n * 2L + 1) * plane + pix] = o[1];
    }
}

// First half of a split drain: from the two grid_change outputs of pixel (y, x) to the four corner loads of its sampling tap,
// nothing else.  The caller keeps `v` in registers, does unrelated work, then calls tail_epilogue(..., &v), which recomputes the
// same tap and blends the loaded corners.  Returns false when this KIND does not sample (decomposer) or no interleaved image exists.
template <int KIND>
__device__ __forceinline__ bool tail_gather_issue(const float (&o)[TAIL_CO_PAD], int n, int y, int x, int S, const float* __restrict__ base,
                                                  const float* __restrict__ g0, int g0_ld, float4 (&v)[4]) {
    if (KIND == TAIL_DECOMPOSER || g0 == nullptr) return false;
    const GsTap t = (KIND == TAIL_UNET) ? gs_locate(base[x], base[y], o[4], o[5], S, S) : gs_locate(base[x], base[y], o[0], o[1], S, S);
    gs_issue4_nhwc(g0 + (size_t)n * S * S * g0_ld, g0_ld, S, S, t, v);
    return true;
}

}  // namespace tha4
