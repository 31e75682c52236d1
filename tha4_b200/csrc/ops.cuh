// Non-GEMM kernels of the THA4 hot path (declarations): normalisation, FiLM, small dense layers, attention,
// image glue (layout change, crop/paste, bilinear resize, grid_sample) and the fused decoder tails.
#pragma once
#include "common.cuh"

namespace tha4 {

// ---------------------------------------------------------------- normalisation (norm.cu)
// Accumulates per-(n,c) sum / sum of squares of x into x.stats (must be zero on entry).  Only needed for tensors whose
// producer did not already do it (the wgmma conv epilogue and the split-K reduction accumulate them for free).
void norm_stats(const View& x, cudaStream_t s);

// Turns the statistics into a per-(n,c) affine  y = x * A + B  that folds InstanceNorm2d / GroupNorm (eps 1e-5,
// biased variance; nn/normalization.py:94-95, unet.py:65-66) with gamma/beta and up to two FiLM scale-shifts
// h*(1+s)+b (unet.py:90-97,159-163).  coef: [N][C][2] floats.
//   groups == 0: instance norm (one group per channel).  film0: [2C] shared by all samples (the t=0 time embedding
//   is a constant); film1: [N][film1_ld] with this block's 2C vector at film1 + n*film1_ld.
void norm_finalize(const View& x, int groups, const float* gamma, const float* beta,
                   const float* film0, const float* film1, int film1_ld, float* coef, cudaStream_t s);
// norm_finalize + norm_apply in one launch: every CTA rebuilds the affine of its sample in shared memory from x.stats.
void norm_apply_fused(const View& x, int groups, const float* gamma, const float* beta, const float* film0,
                      const float* film1, int film1_ld, int act, int pool, const View* res, const View& y, cudaStream_t s,
                      int round_out, const View* y16 = nullptr,    // y may itself be an f16 view; y16: extra f16 copy of an fp32 y
                      const View* xpool = nullptr);                // pool == 1: also the 2x2 mean of the RAW input (fp32), e.g. a down block's skip path

// y = act(x * A + B) (+ res).  pool == 1: y has half the resolution and is the 2x2 mean of the activated values
// (AvgPool2d(2) after SiLU, unet.py:58,158).  x and y may alias when pool == 0.
// round_out: round the result to TF32 (it is a tensor-core operand of the next conv; see round_tf32 in common.cuh).
void norm_apply(const View& x, const float* coef, int act, int pool, const View* res, const View& y, cudaStream_t s,
                int round_out = 0);

// ---------------------------------------------------------------- small dense layers (linear.cu)
// y[n][o] = bias[o] + sum_i f(x[n][i]) * W[o][i],  f = SiLU if silu_in else identity.  x: [N][x_ld], y: [N][y_ld].
void linear_forward(const float* x, int x_ld, int N, int I, const float* W, const float* bias, int O, int silu_in,
                    float* y, int y_ld, cudaStream_t s);

// ---------------------------------------------------------------- attention (attention.cu)
// qkv: NHWC [N,L=H*W,3C] with q|k|v channel blocks ("new order", unet.py:192-202), heads of C/heads channels.
// out: NHWC [N,L,C].  L must be 256, head dim 32.
// fast: the default precision mode may use the tensor-core kernel (f16 operands); strict callers pass false.
void attention_forward(const View& qkv, int heads, const View& out, cudaStream_t s, bool fast = false);
void attention_enable_mma(bool on);       // option "attn_mma" (default on)
void attention_enable_split16(bool on);   // 16 CTAs per (sample, head) instead of 4 (B=1 latency; opt-in)

// ---------------------------------------------------------------- image glue (image_ops.cu)
void nchw_to_nhwc(const ImgView& src, const View& dst, cudaStream_t s);                 // dst.C == src.C
void nhwc_to_nchw(const View& src, float* dst, cudaStream_t s);                          // dst contiguous NCHW
void copy_window(const ImgView& src, float* dst, long dn, long dc, long dh, cudaStream_t s);  // strided NCHW copy
void tile_vector(const float* vec, int vec_ld, int P, const View& dst, cudaStream_t s); // dst[n,y,x,c] = c<P ? vec[n][c] : 0  (dst fp32 or f16)
void convert_f16(const View& src, const View& dst, cudaStream_t s);                      // fp32 view -> f16 view (tests)
void convert_flat_f16(const float* src, __half* dst, long n, cudaStream_t s);               // element-wise, same layout
void convert_flat_f32(const __half* src, float* dst, long n, cudaStream_t s);
void convert_f32(const View& src, const View& dst, cudaStream_t s);                      // f16 view -> fp32 view (tests)
void resize_bilinear(const ImgView& src, float* dst, int Ho, int Wo, cudaStream_t s);   // align_corners=False
void grid_sample(const ImgView& image, const float* grid_change, float* out, int* x0, int* y0, float* tx, float* ty,
                 cudaStream_t s);                                                        // any output may be null
// Upscaler02 prologue (upscaler_02.py:76-80 + mode_07.py:114-115): bilinear x2 of the half-res posed image and
// grid change, warp of the rest image by the coarse grid, all concatenated as NHWC
// [rest(4) | coarse_posed(4) | warped(4) | coarse_grid(2) | 0 0].
// coarse_size: resolution of `posed` / `grid` (S/2 in the fused pipeline; S when the caller already upsampled).
void upscaler_prologue(const ImgView& rest, const float* posed, const float* grid, int coarse_size, const View& dst,
                       cudaStream_t s);
// Its adjoint for dx0, the gradient of dst (NHWC, >= 14 channels; 14, 15 unread): drest (NHWC [N,S,S,4], 4 floats per pixel,
// accumulated into with atomics; null = not wanted) += the rest-image terms (identity + the warp's image adjoint); d_posed
// [N,4,coarse,coarse] / d_grid [N,2,coarse,coarse] (NCHW, overwritten, null = not wanted): the posed / grid terms through the
// bilinear x2 adjoint (a fixed-order gather; the grid gradient of the warp is zero where the border clamp is active).
void upscaler_prologue_backward(const ImgView& rest, const float* grid, int coarse_size, const View& dx0, float* drest,
                                float* d_posed, float* d_grid, cudaStream_t s);
// Poser output [B,4,H,W] in [-1,1] -> [B,H,W,4] uint8 sRGB (+ optional opaque background), and PNG pixels [H,W,4] uint8 ->
// poser input [4,H,W]; see image_ops.cu.
void frame_to_srgb8(const float* frame, int B, int H, int W, int background, int round_mode, unsigned char* out, cudaStream_t s);
void rgba8_to_poser_image(const unsigned char* rgba, int H, int W, float* out, cudaStream_t s);
// max |a - b| > 0 ?  (eyebrow-decomposer cache check, mode_07.py:56-61).  Synchronises the stream.
bool images_differ(const float* a, const float* b, size_t n, int* dev_flag, cudaStream_t s);
// Base-grid table (affine_grid identity, align_corners=False) for a given size; device pointer, cached.
const float* base_grid_table(int size);
void base_grid_host(int W, float* out);

// ---------------------------------------------------------------- fused decoder tails (tail.cu)
enum TailKind { TAIL_UNET = 0, TAIL_DECOMPOSER = 1, TAIL_COMBINER = 2, TAIL_FACE = 3 };
struct TailWeights {
    float* w = nullptr;      // [9][C][CO_PAD] fp32
    float* bias = nullptr;   // [CO_PAD]
    int C = 0, CO = 0;
    __half* w16 = nullptr;   // [9][16][C] f16, K-major B operand of the wgmma tail (tail_make_half), scaled by w16_scale
    float w16_scale = 1.0f;
};
// pending normalisation of the tail's feature map (applied inside the wgmma tail from the feature view's statistics)
struct NormSpecTail { int groups = 0; int act = ACT_NONE; const float* gamma = nullptr; const float* beta = nullptr; };
constexpr int TAIL_CO_PAD = 12;
// Head weights: tail_init allocates zeroed storage (recorded in the active AllocSink), tail_add appends one reference
// head conv (weight [cout, C, 3, 3], bias [cout] or nullptr) in the channel order the kernel expects for its kind.
void tail_init(TailWeights& tw, int C, cudaStream_t s);
void tail_add(TailWeights& tw, const float* w_ref, const float* b_ref, int cout, cudaStream_t s);
// feature: raw conv output NHWC; coef: per-(n,c) affine from norm_finalize; act: ReLU (enc-dec) or SiLU (U-Net).
// image0: the image that is warped / blended (NCHW view); image1: second image (combiner: background layer).
// outputs: NCHW contiguous, order/meaning per kind (see tail.cu).
void tail_forward(TailKind kind, const TailWeights& tw, const View& feature, const float* coef, int act,
                  const ImgView& image0, const ImgView& image1, float* const* outputs, cudaStream_t s, int strict);
// wgmma variant (tail_tc.cu): `feature` is the RAW f16 feature map with the statistics its producer accumulated
void tail_make_half(TailWeights& tw, cudaStream_t s);     // f16 B-operand copy of the head weights (recorded in the active AllocSink)
bool tail_tc_supported(const TailWeights& tw, const View& feature);
void tail_tc_enable_persist(bool on);      // option "tail_persist": persistent pipelined tensor-core tail (default on)
// gather0 / gather1: optional fp32 NHWC copies of image0 / image1 (4-channel slices, 16-byte aligned pixels), e.g. the
// network's own input tensor: the persistent kernel then reads a pixel's RGBA with one 16-byte load (same values, same results)
void tail_tc_forward(TailKind kind, const TailWeights& tw, const View& feature, const NormSpecTail& ns, const ImgView& image0,
                     const ImgView& image1, float* const* outputs, cudaStream_t s, const View* gather0 = nullptr, const View* gather1 = nullptr);

// ---------------------------------------------------------------- backward of the encoder-decoder networks (encdec_backward.cu)
// InstanceNorm2d(affine) (+ReLU) backward: dx = d/dx of y = act(gamma (x - mean) rstd + beta) for the upstream gradient dy.
// x: the RAW input (fp32 or f16) with its statistics; dy / dx fp32.  sums: N*C*2 zeroed doubles of workspace.
void norm_backward(const View& x, const float* gamma, const float* beta, int act, const View& dy, const View& dx, double* sums, cudaStream_t s);
// Tail backward (any kind): from the forward's outputs and their upstream gradients (grads[k] may be null) to dh [N,S,S,16]
// (head pre-activation gradients in the tail's channel order, rest zero) and the image terms: d0 / d1 NHWC with `dld` floats
// per pixel (null = not wanted); d0 must be zero on entry for the warping kinds (U-Net, combiner, face).
void tail_backward(TailKind kind, const float* const* outputs, const float* const* grads, const ImgView& image0, const ImgView& image1,
                   const View& dh, float* d0, float* d1, int dld, cudaStream_t s);

// ---------------------------------------------------------------- backward of the U-Net (unet_backward.cu)
// GroupNorm(groups) (+ FiLM scale-shifts film0 [2C] / film1 [N][film1_ld]) (+ SiLU when act == ACT_SILU) backward, exact SiLU'
// at the recomputed pre-activation.  x: the RAW input (fp32 or f16) with its statistics; dy, dx fp32 at x's resolution, or dy at
// half of it when dy_pool (the layer's output was 2x2-mean-pooled).  dx also gets + res (res_mode RES_SAME, RES_UP2: 2x2 sum of
// a 2x tensor, RES_DOWN2: 1/4 of a half-resolution tensor; conv.cuh) + add (same resolution); either may be null.  dfilm
// (optional, needs film1): d(scale) / d(shift) of film1 into [N][dfilm_ld] at c / C + c.  sums: N*C*2 zeroed doubles;
// coef: N*C*8 floats of workspace.  C <= 512.
void group_norm_backward(const View& x, int groups, const float* gamma, const float* beta, const float* film0, const float* film1,
                         int film1_ld, int act, const View& dy, int dy_pool, const View& dx, float* dfilm, int dfilm_ld,
                         const View* res, int res_mode, const View* add, double* sums, float* coef, cudaStream_t s);
// qkv_attention backward (fp32, deterministic): qkv NHWC [N,256,3C] as attention_forward read it, dout [N,256,C] -> dqkv
// [N,256,3C] (dq | dk | dv).  rowstat: N*heads*256*4 floats of workspace.
void attention_backward(const View& qkv, const View& dout, int heads, const View& dqkv, float* rowstat, cudaStream_t s);
// data gradient of linear_forward: dx[n][k] = SiLU'(pre[n][k]) sum_r dy[n][r] W[r][k] (pre null: no SiLU), W [R][K], fixed
// order in fp64
void linear_backward(const float* dy, int dy_ld, int N, int R, const float* W, int K, const float* pre, int pre_ld, float* dx, int dx_ld,
                     cudaStream_t s);

}  // namespace tha4
