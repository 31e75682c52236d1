// Implicit-GEMM convolution on NHWC activations (fp32, or f16 behind a normalisation layer) -- declarations.
//
// One kernel family covers every dense contraction of the teacher networks:
//   3x3 s1 p1 (nn/conv.py:38-41, unet.py:133,142,454,529), 4x4 s2 p1 downsample (nn/conv.py:141-147),
//   4x4 s2 p1 transposed upsample as 4 output phases of 2x2 taps (nn/conv.py:171-177), 1x1 (unet.py:152,224-225).
// GEMM view: M = output pixels, N = Cout, K = taps * Cin.
#pragma once
#include "common.cuh"

namespace tha4 {

constexpr int CONV_MAX_TAPS = 16;
constexpr int CONV_MAX_PHASES = 4;

enum ResMode { RES_NONE = 0, RES_SAME = 1, RES_UP2 = 2, RES_DOWN2 = 3 };

// Packed weights: [phase][tap][cout_pad][cin_pad] fp32 (+ an f16 copy in the default mode), cin_pad % 32 == 0,
// cout_pad % 32 == 0, zero padded.
struct ConvWeights {
    float* w = nullptr;
    mutable __half* w16 = nullptr;   // same layout in f16, made on first use with f16 activations (conv_tc.cu)
    mutable float w16_scale = 1.0f;  // power of two the f16 copy was multiplied by (max |w| normalised into [0.5, 1): a layer of
                                     // tiny weights would otherwise land in f16's subnormal range); undone on the accumulator
    float* bias = nullptr;      // [cout] or nullptr
    int cin = 0, cout = 0, cin_pad = 0, cout_pad = 0;
    int ntaps = 0, nphase = 1;
    bool dynamic = false;       // weights are rewritten between launches (distillation): never fetch them ahead of the stream order
    bool tf32_rounded = false;  // weights were rounded to TF32 at pack time (non-strict contexts)
    int stride = 1;             // input stride
    int out_mul = 1;            // output coordinate = m * out_mul + phase offset (2 for the transposed conv)
    signed char dy[CONV_MAX_PHASES][CONV_MAX_TAPS];
    signed char dx[CONV_MAX_PHASES][CONV_MAX_TAPS];
    signed char ph_oy[CONV_MAX_PHASES], ph_ox[CONV_MAX_PHASES];
    // A 1x1 convolution folded into this 3x3 one (conv_make_fold): a second K segment, the f16 weights w16b [cout_pad][cin2_pad]
    // at their own scale w16b_scale, read against ConvArgs::in2; bias is the sum of both biases.  cin2 = 0: none.
    int cin2 = 0, cin2_pad = 0;
    __half* w16b = nullptr;
    float w16b_scale = 1.0f;
};

// CONV_UP2_3x3: nearest-neighbour x2 upsample followed by a 3x3 conv (the up-sampling ResBlock, unet.py:46,119-123),
// evaluated on the LOW-resolution input as four output phases of 2x2 taps whose weights are pre-summed at pack time
// (rows/cols of the 3x3 kernel that read the same source pixel are added): 2.25x fewer MACs, no upsampled tensor.
enum ConvKind { CONV_3x3 = 0, CONV_4x4_S2 = 1, CONVT_4x4_S2 = 2, CONV_1x1 = 3, CONV_UP2_3x3 = 4 };

// Fills the tap tables of `cw` for `kind` (no allocation).
void conv_describe(ConvWeights& cw, ConvKind kind, int cin, int cout);

// Packs reference-layout weights (Conv2d: [Cout,Cin,kh,kw]; ConvTranspose2d: [Cin,Cout,kh,kw]) into cw.w
// (device buffer of conv_packed_floats(cw) floats, zero-filled by this call).  `cin_offset` lets two Conv2d
// weights share one packed tensor along Cin (Upscaler02's first_conv + coarse_image_conv).
size_t conv_packed_floats(const ConvWeights& cw);
void conv_pack(const ConvWeights& cw, ConvKind kind, const float* w_ref, int w_cin, int cin_offset, cudaStream_t s);
void conv_set_pack_rounding(bool round_tf32);   // applies to subsequent conv_pack calls (set from the context's strict option)
bool conv_pack_rounding();
// Data gradient of a conv as a conv of the same family (encdec_backward.cu): packs the adjoint of the FORWARD conv `kind`
// (w_ref [cout,cin,k,k], or [cin,cout,4,4] for CONVT_4x4_S2) into cw, a conv from cout to cin channels (cout_kernel > cin:
// zero extra output channels).  3x3 s1 p1 -> 3x3 with W^T flipped; 4x4 s2 conv <-> 4x4 s2 transposed conv, same tensor.
// Allocates cw.w with tracked_malloc; honours conv_pack_rounding().
void conv_pack_adjoint(ConvWeights& cw, ConvKind kind, const float* w_ref, int cin, int cout, int cout_kernel, cudaStream_t s);

// Pending normalisation of the conv's INPUT, applied by the wgmma kernel to its f16 operand tiles in shared memory
// (conv_tc.cu, XF kernels): y = act(A_c x + B_c) with (A, B) built per CTA from the statistics the producing conv
// accumulated -- InstanceNorm2d (groups == 0) / GroupNorm(groups), eps 1e-5, affine, up to two FiLM scale-shifts.
// Replaces a separate normalisation pass (one launch + one read and one write of the tensor) per conv.
struct ConvNormIn {
    bool on = false;
    int C = 0;                  // leading channels of `in` that are normalised (the rest -- tiled pose planes -- pass through)
    int groups = 0, act = ACT_NONE;
    const float* gamma = nullptr; const float* beta = nullptr;
    const float* film0 = nullptr; const float* film1 = nullptr; int film1_ld = 0;
    const double* stats = nullptr; int stats_ld = 0, stats_rep = 1; long stats_rep_stride = 0;   // statistics of the raw input tensor
};

struct ConvArgs {
    View in;                    // stored input (if in_up: stored at half the logical resolution)
    int in_up = 0;              // nearest-neighbour x2 upsample fused into the gather (unet.py:46)
    View out;                   // geometry + statistics slot of the output; out.p may be null when only the f16 copy is wanted
    View out16;                 // optional f16 copy of the output (out16.p == nullptr: none)
    ConvNormIn nin;             // fused normalisation of the input (wgmma kernel, f16 input only)
    View in2;                   // f16 input of a folded 1x1 conv (cw.cin2 > 0), at the output's resolution
    View res;                   // residual added in the epilogue (res.p == nullptr: none)
    int res_mode = RES_NONE;    // RES_UP2: res stored at half resolution; RES_DOWN2: res at double resolution (2x2 mean)
    int strict = 0;             // 1: 3xTF32 error-compensated products (fp32-equivalent); 0: single TF32
    int ksplit = 0;             // 0: choose automatically
    float* ws = nullptr;        // optional split-K workspace (conv_workspace_floats); without it split-K accumulates atomically
    size_t ws_floats = 0;
};

// Floats of workspace the wgmma kernel wants for this call (0: none needed / not the wgmma path).
size_t conv_workspace_floats(const ConvWeights& cw, const ConvArgs& a);

// out = conv(in) + bias (+ res).  When the launch splits K, `out` is zeroed first on the same stream.
// Dispatches to the wgmma kernel (conv_tc.cu) when it supports the configuration, else to the mma.sync kernel.
void conv_forward(const ConvWeights& cw, const ConvArgs& a, cudaStream_t s);
void conv_mma_forward(const ConvWeights& cw, const ConvArgs& a, cudaStream_t s);     // conv.cu (general shapes, strict mode)
bool conv_tc_supported(const ConvWeights& cw, const ConvArgs& a);
void conv_tc_forward(const ConvWeights& cw, const ConvArgs& a, cudaStream_t s);      // conv_tc.cu (wgmma + TMA)
// True when conv_forward(cw, a) will itself accumulate a.out.stats (wgmma epilogue / split-K reduction); otherwise
// the caller runs norm_stats on the output.
bool conv_fuses_stats(const ConvWeights& cw, const ConvArgs& a);
bool conv_tc_fuses_stats(const ConvWeights& cw, const ConvArgs& a);
// How the wgmma kernel would split K for this call: 0 not split (or not the wgmma kernel), 1 over a cluster, 2 through the
// workspace, 3 with atomics into the output (no workspace given)
int conv_tc_split_plan(const ConvWeights& cw, const ConvArgs& a);
// conv_halo.cu: 3x3 stride-1 convs on f16 operands with halo reuse (one activation box per channel chunk, taps as
// row-shifted UMMA descriptors); preferred over conv_tc_forward when it supports the configuration
bool conv_halo_supported(const ConvWeights& cw, const ConvArgs& a);
void conv_halo_forward(const ConvWeights& cw, const ConvArgs& a, cudaStream_t s);
// The halo launch conv_halo_forward(cw, a) would make, from the same plan (false: not the halo kernel).  info[0..6]: N tile
// width, cluster size, consumer warpgroups, resident CTAs per SM, phases, TMA-store bits (1 fp32 out, 2 f16 out, 4 residual
// box), channel chunks
bool conv_halo_plan_info(const ConvWeights& cw, const ConvArgs& a, int* info);
void conv_halo_debug_dump();   // developer: THA4_HALO_DEBUG=1 phase stamps of the last halo launch
void conv_make_half(const ConvWeights& cw, cudaStream_t s);   // f16 copy of the packed weights (cw.w16), recorded in the active AllocSink
// conv3 (3x3) followed by conv1x1 (same Cout) as one K (ConvWeights::cin2): the two f16 copies as they are (not owned by
// `fold`), and the summed bias, recorded in the active AllocSink
void conv_make_fold(ConvWeights& fold, const ConvWeights& conv3, const ConvWeights& conv1x1, cudaStream_t s);

}  // namespace tha4
