// Network assembly for the THA4 hot path: weights in library-owned packed layouts, activations from a caching
// device pool, launch sequences written as plain C++ that reads like the reference forward()s.
#pragma once
#include "common.cuh"
#include "conv.cuh"
#include "ops.cuh"
#include <map>
#include <unordered_map>
#include <memory>
#include <string>
#include <vector>

namespace tha4 {

// Exact-size caching device allocator.  A forward pass requests the same sizes in the same order every time, so
// after the first call no cudaMalloc happens and every buffer keeps its address (CUDA-graph friendly).
class Pool {
public:
    ~Pool();
    float* alloc(size_t nfloats);
    double* alloc_f64(size_t n) { return reinterpret_cast<double*>(alloc(2 * n)); }
    void reset();          // every block becomes reusable (stream order makes reuse safe: one stream per ctx call)
    size_t bytes() const { return total_; }
private:
    struct Bucket { std::vector<void*> blocks; size_t next = 0; };
    std::unordered_map<size_t, Bucket> buckets_;   // O(1) per request: a pass makes ~600 of them between kernel launches
    std::vector<void*> all_;
    size_t total_ = 0;
};

struct TensorRef { const float* p = nullptr; std::vector<long> shape; long numel() const; };
using StateDict = std::map<std::string, TensorRef>;

struct NormW { float* gamma = nullptr; float* beta = nullptr; int C = 0; };

struct Runtime {                      // per-call execution context
    Pool* persist;
    Pool* scratch;
    cudaStream_t stream;
    int strict;
    int f16 = 0;                      // normalisation layers hand f16 tensors to the wgmma convs (non-strict, wgmma on)
    // optional second stream + fork / join events: independent branches of the DAG (the 1x1 skip conv of a ResBlock next to
    // its norm0 -> conv0 chain) run beside the main chain -- also inside a captured graph, where they become parallel branches
    cudaStream_t side = nullptr;
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
    // zero-initialised arena for per-(n,c) statistics (View::stats); bump-allocated, re-zeroed by the caller per pass
    double* stats_base = nullptr;
    size_t stats_cap = 0;
    size_t* stats_off = nullptr;
    double* alloc_stats(size_t n);
};

// ------------------------------------------------------------------ encoder-decoder networks
// The activations a backward pass reads from the forward it recomputes: the NHWC network input and the RAW output of every
// conv that is followed by an InstanceNorm (fp32 or f16 data, with the statistics the producing conv accumulated).
struct EncDecTape {
    View x0;
    View down[4], bott0, res[5][2], up[3];
};

// What EncDecNet::backward computes.  grad_outputs: the upstream gradients of the network's outputs (NCHW, an entry may be
// null = zero).  Every other pointer is an output, null = not computed: d_image0 / d_image1 follow forward()'s image0 /
// image1, d_pose is [N][d_pose_ld] (its first pose_ch entries per row are written).
struct EncDecGrads {
    const float* const* grad_outputs = nullptr;
    float* d_image0 = nullptr;
    float* d_image1 = nullptr;
    float* d_pose = nullptr;
    int d_pose_ld = 0;
};

// EyebrowDecomposer00 / EyebrowMorphingCombiner00 / FaceMorpher08 (poser_encoder_decoder_00.py:43-121,
// face_morpher_08.py:48-202): conv3 + 3 stride-2 convs, bottleneck conv (pose concat) + 5 ResnetBlocks, 3 transposed
// convs, fused head tail.
class EncDecNet {
public:
    EncDecNet(TailKind kind, int size, int in_ch, int pose_ch);
    void load(const StateDict& sd, cudaStream_t s);
    // image0 / image1: see tail.cu (decomposer, face: image1 unused; combiner: image0 = eyebrow layer,
    // image1 = background layer, network input = cat(background, eyebrow)).
    void forward(Runtime& rt, const ImgView& image0, const ImgView& image1, const float* pose, int pose_ld,
                 float* const* outputs, EncDecTape* tape = nullptr);
    // Input gradients (encdec_backward.cu): recomputes the forward in the context's precision mode, keeping its activations,
    // then runs the adjoint of every layer back to the inputs that were asked for.
    void backward(Runtime& rt, const ImgView& image0, const ImgView& image1, const float* pose, int pose_ld, const EncDecGrads& g);
    int size() const { return S_; }
    int num_outputs() const { return kind_ == TAIL_DECOMPOSER ? 6 : 8; }
    bool loaded() const { return loaded_; }
private:
    void forward_fused(Runtime& rt, const View& x0, const ImgView& image0, const ImgView& image1, const float* pose, int pose_ld,
                       float* const* outputs, EncDecTape* tape);
    void load_adjoints(const StateDict& sd, const std::string& prefix, cudaStream_t s);
    AllocSink owned_;          // every device allocation made by load()
    TailKind kind_;
    int S_, in_ch_, pose_ch_, pose_pad_;
    bool loaded_ = false;
    ConvWeights down_[4], bott0_, res_[5][2], up_[3];
    NormW down_n_[4], bott0_n_, res_n_[5][2], up_n_[3];
    TailWeights tail_;
    // adjoint-packed weights (data gradients on the same conv kernels): 3x3 -> 3x3 with W^T flipped, 4x4 s2 <-> transposed
    ConvWeights adj_down_[4], adj_bott0_, adj_res_[5][2], adj_up_[3], adj_head_;
};

// ------------------------------------------------------------------ U-Net networks
struct ResBlockW {
    int cin = 0, cout = 0;
    NormW norm0, norm1;
    ConvWeights conv0, conv1, skip;
    bool has_skip = false;
    float* film0 = nullptr;     // [2*cout], constant (t = 0 time embedding, unet.py:365-376)
    int film1_off = 0;          // offset of this block's 2*cout FiLM vector in the batched pose projection
};
struct AttnW { int C = 0; NormW norm; ConvWeights qkv, proj; };

// The activations the U-Net backward reads from the forward it recomputes, keyed by the block's weights (each block runs
// once per forward).  Normalised tensors are kept as the normalisation read them (fp32, or the f16 operand copy), with the
// statistics their producer accumulated.
struct UNetTape {
    struct Res { View x, h0; };       // block input (norm0), raw conv0 output (norm1)
    struct Attn { View x, qkv; };     // block input (norm), qkv projection (fp32)
    std::map<const ResBlockW*, Res> res;
    std::map<const AttnW*, Attn> attn;
    const float* c1 = nullptr;        // pose MLP pre-activations [N][256] (unet.py:449-452): cond_embed.0 output
    const float* c2 = nullptr;        //   cond_embed.2 output
    const float* film1 = nullptr;     // the batched pose FiLM table [N][film1_total]
    View feat;                        // last feature map (last.0's input)
};

// What UNetNet::backward computes: grad_outputs[5] (merged, alpha, warped, grid_change, direct; NCHW, null = zero);
// d_image [N,4,S,S] (the upscaler: its rest image), d_pose [N][d_pose_ld] (first 6 entries per row) and, on the upscaler only,
// d_coarse_posed [N,4,c,c] / d_coarse_grid [N,2,c,c] (c = coarse_size) are outputs, null = not computed.
struct UNetGrads {
    const float* const* grad_outputs = nullptr;
    float* d_image = nullptr;
    float* d_pose = nullptr;
    int d_pose_ld = 0;
    float* d_coarse_posed = nullptr;
    float* d_coarse_grid = nullptr;
};

// Frames per pass of the upscaler backward.  Its taped forward and gradient buffers at 512x512 take 2610 MiB of the context's
// workspace pool per frame (measured on an H100 at B = 1 and 2, DESIGN.md section 4), and the pool keeps its peak: 6 frames
// keep a pass under 16 GiB.
constexpr int UPSCALER_BWD_MAX_BATCH = 6;

// Morpher00 (morpher_00.py:35-72) and Upscaler02 (upscaler_02.py:37-102) on Unet / UnetWithFirstConvAddition
// (unet.py:438-546,549-658).
class UNetNet {
public:
    UNetNet(bool upscaler, int size, int model_channels, std::vector<int> mults);
    void load(const StateDict& sd, cudaStream_t s);
    // morpher: image = [B,4,S,S]; upscaler: image = rest image, half_posed / half_grid at S/2 (mode_07.py:111-118).
    // tape: keep what backward() reads (its tensors then live in rt.persist; normalisations write out of place).
    void forward(Runtime& rt, const ImgView& image, const float* coarse_posed, const float* coarse_grid, int coarse_size,
                 const float* pose, int pose_ld, float* const* outputs, UNetTape* tape = nullptr);
    // Input gradients (unet_backward.cu): recomputes the forward (same inputs as forward()) in the context's precision mode
    // with a tape, then runs the adjoint of every layer back to the inputs that were asked for.
    void backward(Runtime& rt, const ImgView& image, const float* coarse_posed, const float* coarse_grid, int coarse_size,
                  const float* pose, int pose_ld, const UNetGrads& g);
    int size() const { return S_; }
    bool loaded() const { return loaded_; }
private:
    AllocSink owned_;          // every device allocation made by load()
    void forward_fused(Runtime& rt, const ImgView& image, const float* coarse_posed, const float* coarse_grid, int coarse_size,
                       const float* pose, int pose_ld, float* const* outputs, UNetTape* tape);
    void res_block(Runtime& rt, const ResBlockW& w, const View& x, int mode, const float* film1, const View& out, UNetTape* tape);
    void attn_block(Runtime& rt, const AttnW& w, const View& x, const View& out, UNetTape* tape);
    // adjoint-packed weights, made from the packed forward weights by the first backward() (inference-only contexts never
    // hold them): per ResBlock conv0 / conv1 / skip, per attention block qkv / proj, the first conv and the last.2 head
    struct ResAdj { ConvWeights conv0, conv1, skip; };
    struct AttnAdj { ConvWeights qkv, proj; };
    void pack_adjoints(Runtime& rt);
    bool adj_ready_ = false;
    std::map<const ResBlockW*, ResAdj> adj_res_;
    std::map<const AttnW*, AttnAdj> adj_attn_;
    ConvWeights adj_first_, adj_head_;
    bool upscaler_;
    int S_, mc_, L_;
    std::vector<int> mults_;
    bool loaded_ = false;
    ConvWeights first_;
    std::vector<ResBlockW> down_res_, down_ds_, mid_res_, up_res_, up_us_;   // up_res_: 2 per level
    std::vector<AttnW> mid_attn_, up_attn_;
    AttnW down_attn_;
    float *cond_w0_ = nullptr, *cond_b0_ = nullptr, *cond_w2_ = nullptr, *cond_b2_ = nullptr;
    float *film1_w_ = nullptr, *film1_b_ = nullptr;
    int film1_total_ = 0;
    NormW last_n_;
    TailWeights tail_;
};

// ------------------------------------------------------------------ backward helpers shared by the networks
// Data gradient of a conv on the conv kernels: dx = conv(dy) with adjoint-packed weights (+ add, same resolution).
void run_dgrad(Runtime& rt, const ConvWeights& cw, const View& dy, const View& dx, const View* add = nullptr);
// The fused tail's head conv (tw.w) as one packed 3x3 conv from its 16-channel head-gradient tensor to the tw.C features.
void head_pack_adjoint(ConvWeights& cw, const TailWeights& tw, bool round_w, cudaStream_t s);
// adjoint of a PACKED forward conv (fwd, of kind `kind`) as a conv from fwd.cout to fwd.cin channels: 3x3 -> 3x3 with W^T
// flipped, 1x1 -> 1x1 with W^T, CONV_UP2_3x3 (nearest x2 + 3x3, pre-summed phases) -> 4x4 stride-2 conv with W^T.  Allocates
// cw.w with tracked_malloc; the values are those of fwd (TF32-rounded iff fwd's are).
void conv_adjoint_from_packed(ConvWeights& cw, const ConvWeights& fwd, ConvKind kind, cudaStream_t s);

}  // namespace tha4
