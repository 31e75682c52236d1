// Weight-gradient convolution of the teacher networks (conv_wgrad.cu) -- declarations.
#pragma once
#include "common.cuh"
#include "conv.cuh"
#include <functional>

namespace tha4 {

// Operand transform of a weight-gradient operand: the value the forward conv multiplied, from what the tape keeps.
enum WgradXf {
    WG_XF_NONE = 0,        // the stored value (fp32, or f16 widened)
    WG_XF_HALF = 1,        // f16 FMA with f16-rounded coefficients (the forward's fused normalisation, wgrad_xf_coef)
    WG_XF_FLOAT = 2,       // fp32 FMA (the strict tail's normalisation, coefficients from norm_finalize)
    WG_XF_FLOAT16 = 3,     // fp32 FMA rounded to f16 (the default-mode tail's operand)
};

// An NHWC operand: `C` channels are read (ld elements per pixel), f16 or fp32; channels < coef_C get y = act(A x + B) with
// coef[n][c] = (A, B); the rest pass through (pose planes).  act (Act):
//   ACT_RELU       max(y, 0) in the transform's precision;
//   ACT_SILU       fp32 y / (1 + expf(-y)) (WG_XF_FLOAT: the strict tail);
//   ACT_SILU_FAST  h + h tanh(h) with h = y / 2 -- WG_XF_HALF: in f16 with tanh.approx.f16x2 on coefficients that hold A / 2,
//                  B / 2 already (the wgmma convs' operand transform, conv_tc_device.cuh); WG_XF_FLOAT / WG_XF_FLOAT16: fp32
//                  with tanh.approx.f32, the halving done here (the wgmma tail, tail_tc.cu).
struct WgradOperand {
    const void* p = nullptr;
    int f16 = 0, ld = 0;
    int N = 0, H = 0, W = 0, C = 0;
    int xf = WG_XF_NONE, act = ACT_NONE;
    const float2* coef = nullptr;
    int coef_C = 0;
};

// The operand that reads View v as stored (no transform).
inline WgradOperand wgrad_operand(const View& v) {
    WgradOperand o;
    o.p = v.p; o.f16 = v.f16; o.ld = v.ld; o.N = v.N; o.H = v.H; o.W = v.W; o.C = v.C;
    return o;
}

// dW[d][c][tap] (+)= sum_p D[p][d] G[p * stride - pad + (ky, kx)][c], tap = ky * ksz + kx, written to out at
// out_row[d] + c * ntaps + tap (n_map > 0: rows d >= n_map are dropped), else at (d * c_real + c) * ntaps + tap; channels
// c >= c_real of G are not written.  accumulate: add to what out holds (later micro-batch chunks).
struct WgradArgs {
    WgradOperand G, D;
    int ksz = 3, ntaps = 9, stride = 1, pad = 1;
    int M = 0;                         // ntaps * G.C
    int c_real = 0;
    float* out = nullptr;
    long out_row[16] = {};
    int n_map = 0;
    int accumulate = 0;
    // filled by conv_wgrad from the plan
    int kblocks = 0, kb_per_split = 0, splits = 1;
    float* ws = nullptr; int ws_rows = 0, ws_cols = 0;
    int up2 = 0;                       // G is read through a nearest x2 up-sampling: tap (y + ky - 1, x + kx - 1) is checked at D's
                                       // resolution, then halved (CONV_UP2_3x3)
};

// How a launch is cut: nt output columns per CTA (16 / 64 / 128), 64-row tiles, pixel blocks of 32 split over `splits`
// CTAs (only when the tiles alone cannot fill the GPU twice over), summed from a workspace in split order.
struct WgradPlan { int nt = 0, mtiles = 0, ntiles = 0, kblocks = 0, kb_per_split = 0, splits = 1; };

WgradPlan conv_wgrad_plan(const WgradArgs& a, int ksplit = 0);
size_t conv_wgrad_workspace_floats(const WgradPlan& pl);
void conv_wgrad(WgradArgs a, const WgradPlan& pl, int strict, float* ws, cudaStream_t s);
// The weight gradient of one conv of `kind` (CONV_3x3, CONV_1x1, CONV_UP2_3x3, CONV_4x4_S2, CONVT_4x4_S2) from the operand
// x^ the forward multiplied and the gradient dz at its raw output, as the network backward runs it: Conv2d G = x^, D = dz;
// ConvTranspose2d G = dz, D = x^; nearest x2 + 3x3: x^ at half D's resolution.  `a` carries the destination (out, out_row / n_map, c_real (0: every channel of G), accumulate); ksplit > 0 forces
// the pixel split; ws_alloc hands out the split workspace.  Returns the plan that ran.
WgradPlan conv_wgrad_layer(ConvKind kind, const WgradOperand& x, const WgradOperand& dz, WgradArgs a, int strict, int ksplit,
                           const std::function<float*(size_t)>& ws_alloc, cudaStream_t s);
// coef[n][c] = the (A, B) of the pending InstanceNorm (groups == 0) or GroupNorm (+ FiLM0 [2C] + FiLM1 row n of film1, ld
// film1_ld) (+act) of `raw` (its statistics), built by the forward's fused-normalisation code (xf_build_coef) and rounded to
// f16 as it rounds them (SiLU: A / 2, B / 2); C channels, coef holds raw.N * C float2
float2* wgrad_xf_coef(const View& raw, const float* gamma, const float* beta, int C, int act, float2* coef, cudaStream_t s,
                      int groups = 0, const float* film0 = nullptr, const float* film1 = nullptr, int film1_ld = 0);

}  // namespace tha4
