// Network assembly: weight loading / packing and the launch sequences of the five teacher networks.
#include "nets.cuh"
#include <algorithm>
#include <cmath>
#include <cstdlib>

namespace tha4 {

// ------------------------------------------------------------------------------------------------ Pool
Pool::~Pool() { for (void* p : all_) cudaFree(p); }

float* Pool::alloc(size_t nfloats) {
    size_t bytes = ((nfloats * sizeof(float) + 255) / 256) * 256;
    if (bytes == 0) bytes = 256;
    Bucket& bk = buckets_[bytes];                 // blocks of this exact size, handed out in creation order
    if (bk.next < bk.blocks.size()) return reinterpret_cast<float*>(bk.blocks[bk.next++]);
    void* p = nullptr;
    THA4_CUDA_CHECK(cudaMalloc(&p, bytes));
    bk.blocks.push_back(p);
    bk.next = bk.blocks.size();
    all_.push_back(p);
    total_ += bytes;
    return reinterpret_cast<float*>(p);
}

void Pool::reset() { for (auto& kv : buckets_) kv.second.next = 0; }

long TensorRef::numel() const { long n = 1; for (long d : shape) n *= d; return n; }

double* Runtime::alloc_stats(size_t n) {
    THA4_REQUIRE(stats_base != nullptr && stats_off != nullptr, "statistics arena not set up");
    const size_t off = *stats_off;
    THA4_REQUIRE(off + n <= stats_cap, "statistics arena exhausted (lower the micro-batch)");
    *stats_off = off + n;
    return stats_base + off;
}

// ------------------------------------------------------------------------------------------------ helpers
namespace {

const TensorRef& sd_get(const StateDict& sd, const std::string& key) {
    auto it = sd.find(key);
    if (it == sd.end()) throw std::runtime_error("tha4: state_dict is missing key '" + key + "'");
    return it->second;
}

float* dev_alloc(size_t n) { return reinterpret_cast<float*>(tracked_malloc(std::max<size_t>(n, 1) * sizeof(float))); }   // owned by the loading net

float* dev_clone(const TensorRef& t, cudaStream_t s) {
    float* p = dev_alloc(t.numel());
    THA4_CUDA_CHECK(cudaMemcpyAsync(p, t.p, t.numel() * sizeof(float), cudaMemcpyDeviceToDevice, s));
    return p;
}

NormW load_norm(const StateDict& sd, const std::string& prefix, cudaStream_t s) {
    NormW n;
    const TensorRef& g = sd_get(sd, prefix + ".weight");
    n.C = (int)g.numel();
    n.gamma = dev_clone(g, s);
    n.beta = dev_clone(sd_get(sd, prefix + ".bias"), s);
    return n;
}

// cin_kernel: channel count of the activation tensor the kernel will read (>= the reference Cin, multiple of 4).
ConvWeights load_conv(const StateDict& sd, const std::string& prefix, ConvKind kind, bool bias, cudaStream_t s,
                      int cin_kernel = 0) {
    const TensorRef& w = sd_get(sd, prefix + ".weight");
    THA4_REQUIRE(w.shape.size() == 4, "conv weight rank: " + prefix);
    const int cout = (int)(kind == CONVT_4x4_S2 ? w.shape[1] : w.shape[0]);
    const int cin = (int)(kind == CONVT_4x4_S2 ? w.shape[0] : w.shape[1]);
    const int k = (kind == CONV_3x3 || kind == CONV_UP2_3x3) ? 3 : (kind == CONV_1x1 ? 1 : 4);
    THA4_REQUIRE(w.shape[2] == k && w.shape[3] == k, "conv kernel size: " + prefix);
    ConvWeights cw;
    conv_describe(cw, kind, cin_kernel > 0 ? cin_kernel : cin, cout);
    THA4_REQUIRE(cw.cin >= cin && cw.cin % 4 == 0, "conv cin: " + prefix);
    cw.w = dev_alloc(conv_packed_floats(cw));
    THA4_CUDA_CHECK(cudaMemsetAsync(cw.w, 0, conv_packed_floats(cw) * sizeof(float), s));
    conv_pack(cw, kind, w.p, cin, 0, s);
    cw.tf32_rounded = conv_pack_rounding();
    if (cw.tf32_rounded) conv_make_half(cw, s);      // default mode: most convs read f16 activations (owned by the loading net)
    if (bias) cw.bias = dev_clone(sd_get(sd, prefix + ".bias"), s);
    return cw;
}

void tail_add_head(TailWeights& tw, const StateDict& sd, const std::string& prefix, bool bias, cudaStream_t s) {
    const TensorRef& w = sd_get(sd, prefix + ".weight");
    THA4_REQUIRE(w.shape.size() == 4 && w.shape[1] == tw.C && w.shape[2] == 3 && w.shape[3] == 3, "head shape: " + prefix);
    const int cout = (int)w.shape[0];
    const float* b = bias ? sd_get(sd, prefix + ".bias").p : nullptr;
    tail_add(tw, w.p, b, cout, s);
}

__global__ void vec_add_kernel(float* dst, const float* a, const float* b, int n) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dst[i] = a[i] + b[i];
}

// Replicas of a tensor's statistics slot: producers spread their atomics over them, every consumer CTA folds all of them
// (conv_tc_device.cuh: xf_build_coef).  Developer knob THA4_STATS_REP_MAX (default 16) bounds the count.
int stats_rep_cap() {
    static int cap = [] { const char* e = getenv("THA4_STATS_REP_MAX"); const int v = e ? atoi(e) : 16; return v < 1 ? 1 : (v > 16 ? 16 : v); }();
    return cap;
}

// gives `v` (its geometry set) a zeroed statistics slot: replicas ~ tiles/16 (128-pixel conv tiles per sample), a power of
// two in [1, stats_rep_cap()]
void add_stats(View& v, Runtime& rt) {
    const int tiles = ((v.W + 15) / 16) * ((v.H + 7) / 8);
    int rep = 1;
    while (rep < stats_rep_cap() && rep * 32 <= tiles) rep *= 2;
    v.stats_rep = rep;
    v.stats_rep_stride = (long)v.N * v.C * 2;
    v.stats = rt.alloc_stats((size_t)rep * v.N * v.C * 2);
    v.stats_ld = v.C;
}

// `data` with the statistics slot of `slot`, another view of the same tensor
View with_stats(View data, const View& slot) {
    data.stats = slot.stats; data.stats_ld = slot.stats_ld; data.stats_rep = slot.stats_rep; data.stats_rep_stride = slot.stats_rep_stride;
    return data;
}

}  // namespace

View make_view(Pool* pool, int N, int H, int W, int C, Runtime* rt) {
    View v; v.N = N; v.H = H; v.W = W; v.C = C; v.ld = C;
    v.p = pool->alloc((size_t)N * H * W * C);
    if (rt) add_stats(v, *rt);
    return v;
}

namespace {

// f16 activation tensor (conv operand produced by a normalisation layer; see View::f16)
View make_view16(Pool* pool, int N, int H, int W, int C) {
    THA4_REQUIRE(C % 8 == 0, "f16 view: channels must be a multiple of 8");
    View v; v.N = N; v.H = H; v.W = W; v.C = C; v.ld = C; v.f16 = 1;
    v.p = pool->alloc(((size_t)N * H * W * C + 1) / 2);
    return v;
}

// per-(n,c) affine for the fused tail kernels (InstanceNorm when groups == 0, GroupNorm otherwise)
float* tail_coef(Runtime& rt, const View& x, const NormW& nw, int groups) {
    THA4_REQUIRE(nw.C == x.C, "norm: channel mismatch");
    float* coef = rt.scratch->alloc((size_t)x.N * x.C * 2);
    norm_finalize(x, groups, nw.gamma, nw.beta, nullptr, nullptr, 0, coef, rt.stream);
    return coef;
}

// normalisation layer = one elementwise pass: affine from x.stats rebuilt per CTA, activation / pool / residual fused
void run_norm(Runtime& rt, const View& x, const NormW& nw, int groups, const float* film0, const float* film1,
              int film1_ld, int act, int pool, const View* res, const View& y, const View* y16 = nullptr, const View* xpool = nullptr) {
    THA4_REQUIRE(nw.C == x.C, "norm: channel mismatch");
    norm_apply_fused(x, groups, nw.gamma, nw.beta, film0, film1, film1_ld, act, pool, res, y, rt.stream, !rt.strict, y16, xpool);
}

void run_conv(Runtime& rt, const ConvWeights& cw, const View& in, const View& out, int in_up = 0,
              const View* res = nullptr, int res_mode = RES_NONE) {
    ConvArgs a;
    a.in = in; a.in_up = in_up; a.out = out; a.strict = rt.strict;
    if (res) { a.res = *res; a.res_mode = res_mode; }
    const size_t ws = conv_workspace_floats(cw, a);
    if (ws) { a.ws = rt.scratch->alloc(ws); a.ws_floats = ws; }
    const bool fused = conv_fuses_stats(cw, a);
    conv_forward(cw, a, rt.stream);
    if (out.stats && !fused) norm_stats(out, rt.stream);      // mma.sync path (strict mode, stride-2 convs)
}

// ---- default (tensor-core) mode: activations in up to two precisions, normalisations fused into the consumer conv ----
// An activation tensor as the default mode stores it: `f` always carries the geometry and the statistics slot; f.p is the
// fp32 copy (residual streams, inputs of the few remaining normalisation passes) or null; h is the f16 copy (the operand
// a wgmma conv loads by TMA) or empty.  RAW conv outputs whose only consumer is a conv with a pending normalisation
// exist in f16 only.
struct Tens { View f; View h; };

Tens make_act(Pool* pool, Runtime& rt, int N, int H, int W, int C, bool want_f32, bool want_f16, bool stats = true) {
    Tens a;
    if (want_f32) a.f = make_view(pool, N, H, W, C);
    else { a.f.N = N; a.f.H = H; a.f.W = W; a.f.C = C; a.f.ld = C; }
    if (stats) add_stats(a.f, rt);
    if (want_f16) a.h = make_view16(pool, N, H, W, C);
    return a;
}
// `a` without its fp32 copy (geometry and statistics slot kept): a conv writing it stores the f16 copy and the statistics
// only.  For tensors whose consumers read the data in f16 and the fp32 copy's statistics only.
Tens f16_only(Tens a) { a.f.p = nullptr; return a; }
Tens slice_act(const Tens& a, int c0, int c) {
    Tens r;
    if (a.f.p) r.f = a.f.slice(c0, c);
    else { r.f = a.f; r.f.C = c; if (r.f.stats) r.f.stats = a.f.stats + 2 * c0; }
    if (a.h.p) r.h = a.h.slice(c0, c);
    return r;
}

// the data (fp32 copy if there is one, else the f16 copy) and the statistics slot of a raw conv output
View raw_view(const Tens& a) { return a.f.p ? a.f : with_stats(a.h, a.f); }

// pending normalisation of `src` (its statistics) with the weights of the layer that follows it in the reference graph
ConvNormIn norm_in(const View& src_stats, const NormW& nw, int groups, int act, const float* film0 = nullptr,
                   const float* film1 = nullptr, int film1_ld = 0, int C = 0) {
    THA4_REQUIRE(src_stats.stats != nullptr, "fused normalisation: the producer did not accumulate statistics");
    ConvNormIn n;
    n.on = true; n.C = C > 0 ? C : src_stats.C; n.groups = groups; n.act = act;
    THA4_REQUIRE(nw.C == n.C, "fused normalisation: channel mismatch");
    n.gamma = nw.gamma; n.beta = nw.beta; n.film0 = film0; n.film1 = film1; n.film1_ld = film1_ld;
    n.stats = src_stats.stats; n.stats_ld = src_stats.stats_ld; n.stats_rep = src_stats.stats_rep; n.stats_rep_stride = src_stats.stats_rep_stride;
    return n;
}

// conv on the wgmma kernel: `in` is an f16 operand view (or fp32 for the first layer of a network), `nin` its pending
// normalisation (nullptr: none), `out` receives the fp32 and / or f16 copies it has storage for, plus statistics
// (in2: the f16 input of a folded 1x1 conv, cw.cin2 > 0)
void run_conv_tc(Runtime& rt, const ConvWeights& cw, const View& in, const ConvNormIn* nin, const Tens& out,
                 const View* res = nullptr, int res_mode = RES_NONE, const View* in2 = nullptr) {
    ConvArgs a;
    a.in = in; a.out = out.f; a.out16 = out.h; a.strict = 0;
    if (in2) a.in2 = *in2;
    if (nin) a.nin = *nin;
    if (res) { a.res = *res; a.res_mode = res_mode; }
    const size_t ws = conv_workspace_floats(cw, a);
    if (ws) { a.ws = rt.scratch->alloc(ws); a.ws_floats = ws; }
    THA4_REQUIRE(!out.f.stats || conv_fuses_stats(cw, a), "conv: statistics must be fused on the tensor-core path");
    conv_forward(cw, a, rt.stream);
}

}  // namespace

// ------------------------------------------------------------------------------------------------ EncDecNet
EncDecNet::EncDecNet(TailKind kind, int size, int in_ch, int pose_ch)
    : kind_(kind), S_(size), in_ch_(in_ch), pose_ch_(pose_ch), pose_pad_(round_up(pose_ch, 8)) {}

void EncDecNet::load(const StateDict& sd, cudaStream_t s) {
    SinkScope own(&owned_);
    const std::string p = (kind_ == TAIL_FACE) ? "" : "body.";
    prefix_ = p;
    down_[0] = load_conv(sd, p + "downsample_blocks.0.0", CONV_3x3, false, s);
    down_n_[0] = load_norm(sd, p + "downsample_blocks.0.1", s);
    for (int i = 1; i < 4; ++i) {
        down_[i] = load_conv(sd, p + "downsample_blocks." + std::to_string(i) + ".0", CONV_4x4_S2, false, s);
        down_n_[i] = load_norm(sd, p + "downsample_blocks." + std::to_string(i) + ".1", s);
    }
    bott0_ = load_conv(sd, p + "bottleneck_blocks.0.0", CONV_3x3, false, s, 512 + pose_pad_);
    bott0_n_ = load_norm(sd, p + "bottleneck_blocks.0.1", s);
    for (int i = 0; i < 5; ++i) {
        const std::string rp = p + "bottleneck_blocks." + std::to_string(i + 1) + ".resnet_path.";
        res_[i][0] = load_conv(sd, rp + "0", CONV_3x3, false, s);
        res_n_[i][0] = load_norm(sd, rp + "1", s);
        res_[i][1] = load_conv(sd, rp + "3", CONV_3x3, false, s);
        res_n_[i][1] = load_norm(sd, rp + "4", s);
    }
    for (int i = 0; i < 3; ++i) {
        up_[i] = load_conv(sd, p + "upsample_blocks." + std::to_string(i) + ".0", CONVT_4x4_S2, false, s);
        up_n_[i] = load_norm(sd, p + "upsample_blocks." + std::to_string(i) + ".1", s);
    }
    tail_init(tail_, 64, s);
    if (kind_ == TAIL_DECOMPOSER) {           // packing order expected by tail.cu
        tail_add_head(tail_, sd, "background_layer_alpha.0", true, s);
        tail_add_head(tail_, sd, "background_layer_color_change.0", true, s);
        tail_add_head(tail_, sd, "eyebrow_layer_alpha.0", true, s);
        tail_add_head(tail_, sd, "eyebrow_layer_color_change.0", true, s);
    } else if (kind_ == TAIL_COMBINER) {
        tail_add_head(tail_, sd, "morphed_eyebrow_layer_grid_change", false, s);
        tail_add_head(tail_, sd, "morphed_eyebrow_layer_alpha.0", true, s);
        tail_add_head(tail_, sd, "morphed_eyebrow_layer_color_change.0", true, s);
        tail_add_head(tail_, sd, "combine_alpha.0", true, s);
    } else {
        tail_add_head(tail_, sd, "iris_mouth_grid_change", false, s);
        tail_add_head(tail_, sd, "iris_mouth_color_change.0", true, s);
        tail_add_head(tail_, sd, "iris_mouth_alpha.0", true, s);
        tail_add_head(tail_, sd, "eye_color_change.0", true, s);
        tail_add_head(tail_, sd, "eye_alpha.0", true, s);
    }
    if (conv_pack_rounding()) tail_make_half(tail_, s);       // default mode: the wgmma tail's f16 head weights
    // the flat parameter-gradient layout: the reference's state_dict order (registration order of the modules: per block its
    // conv weight, then the InstanceNorm's weight and bias; then the heads in the tail's packing order, weight then bias)
    head_key_.clear(); head_cout_.clear();
    if (kind_ == TAIL_DECOMPOSER) head_key_ = {"background_layer_alpha.0", "background_layer_color_change.0", "eyebrow_layer_alpha.0", "eyebrow_layer_color_change.0"};
    else if (kind_ == TAIL_COMBINER) head_key_ = {"morphed_eyebrow_layer_grid_change", "morphed_eyebrow_layer_alpha.0", "morphed_eyebrow_layer_color_change.0", "combine_alpha.0"};
    else head_key_ = {"iris_mouth_grid_change", "iris_mouth_color_change.0", "iris_mouth_alpha.0", "eye_color_change.0", "eye_alpha.0"};
    params_ = ParamLayout();
    auto reg_block = [&](const std::string& conv, const std::string& norm) {
        params_.add(sd, conv + ".weight"); params_.add(sd, norm + ".weight"); params_.add(sd, norm + ".bias");
    };
    for (int i = 0; i < 4; ++i) reg_block(p + "downsample_blocks." + std::to_string(i) + ".0", p + "downsample_blocks." + std::to_string(i) + ".1");
    reg_block(p + "bottleneck_blocks.0.0", p + "bottleneck_blocks.0.1");
    for (int i = 0; i < 5; ++i) {
        const std::string rp = p + "bottleneck_blocks." + std::to_string(i + 1) + ".resnet_path.";
        reg_block(rp + "0", rp + "1");
        reg_block(rp + "3", rp + "4");
    }
    for (int i = 0; i < 3; ++i) reg_block(p + "upsample_blocks." + std::to_string(i) + ".0", p + "upsample_blocks." + std::to_string(i) + ".1");
    for (const std::string& h : head_key_) {
        params_.add(sd, h + ".weight");
        head_cout_.push_back((int)sd_get(sd, h + ".weight").shape[0]);
        if (sd.count(h + ".bias")) params_.add(sd, h + ".bias");
    }
    load_adjoints(sd, p, s);
    THA4_CUDA_CHECK(cudaStreamSynchronize(s));
    loaded_ = true;
}

void EncDecNet::forward(Runtime& rt, const ImgView& image0, const ImgView& image1, const float* pose, int pose_ld,
                        float* const* outputs, EncDecTape* tape) {
    THA4_REQUIRE(loaded_, "network weights not loaded");
    THA4_REQUIRE(image0.H == S_ && image0.W == S_ && image0.C == 4, "encdec: image size");
    const int B = image0.N;
    cudaStream_t s = rt.stream;
    Pool* P = rt.persist;
    rt.scratch->reset();

    View x0 = make_view(P, B, S_, S_, in_ch_);
    if (kind_ == TAIL_COMBINER) {   // cat([background_layer, eyebrow_layer], dim=1)  (eyebrow_morphing_combiner_00.py:48)
        nchw_to_nhwc(image1, x0.slice(0, 4), s);
        nchw_to_nhwc(image0, x0.slice(4, 4), s);
    } else {
        nchw_to_nhwc(image0, x0, s);
    }
    if (tape) tape->x0 = x0;
    if (rt.f16) { forward_fused(rt, x0, image0, image1, pose, pose_ld, outputs, tape); return; }
    // conv -> InstanceNorm -> ReLU; the activated tensor goes to `dst`, or back in place (out of place when a backward keeps
    // the raw output: `keep`)
    auto conv_in_relu = [&](const ConvWeights& cw, const NormW& nw, const View& in, int oh, const View* dst, View* keep) -> View {
        View raw = make_view(P, B, oh, oh, cw.cout, &rt);
        run_conv(rt, cw, in, raw);
        const View y = dst ? *dst : (keep ? make_view(P, B, oh, oh, cw.cout) : raw);
        run_norm(rt, raw, nw, 0, nullptr, nullptr, 0, ACT_RELU, 0, nullptr, y);
        if (keep) *keep = raw;
        return y;
    };
    View f = conv_in_relu(down_[0], down_n_[0], x0, S_, nullptr, tape ? &tape->down[0] : nullptr);
    if (tape) { tape->op_down[0] = x0; tape->op_down[1] = f; }
    f = conv_in_relu(down_[1], down_n_[1], f, S_ / 2, nullptr, tape ? &tape->down[1] : nullptr);
    if (tape) tape->op_down[2] = f;
    f = conv_in_relu(down_[2], down_n_[2], f, S_ / 4, nullptr, tape ? &tape->down[2] : nullptr);
    if (tape) tape->op_down[3] = f;
    const int b = S_ / 8;
    View bin = make_view(P, B, b, b, 512 + pose_pad_);
    View bfeat = bin.slice(0, 512);
    conv_in_relu(down_[3], down_n_[3], f, b, &bfeat, tape ? &tape->down[3] : nullptr);
    if (pose_pad_ > 0) tile_vector(pose, pose_ld, pose_ch_, bin.slice(512, pose_pad_), s);   // poser_encoder_decoder_00.py:110-113
    View x = make_view(P, B, b, b, bott0_.cout, &rt);
    run_conv(rt, bott0_, bin, x);
    if (tape) tape->op_bott0 = bin;
    {
        const View y = tape ? make_view(P, B, b, b, bott0_.cout) : x;
        run_norm(rt, x, bott0_n_, 0, nullptr, nullptr, 0, ACT_RELU, 0, nullptr, y);
        if (tape) tape->bott0 = x;
        x = y;
    }
    for (int i = 0; i < 5; ++i) {   // ResnetBlock: x + IN(conv(relu(IN(conv(x)))))  (resnet_block.py:52-67)
        View h = conv_in_relu(res_[i][0], res_n_[i][0], x, b, nullptr, tape ? &tape->res[i][0] : nullptr);
        if (tape) { tape->op_res[i][0] = x; tape->op_res[i][1] = h; }
        View raw = make_view(P, B, b, b, 512, &rt);
        run_conv(rt, res_[i][1], h, raw);
        const View y = tape ? make_view(P, B, b, b, 512) : raw;
        run_norm(rt, raw, res_n_[i][1], 0, nullptr, nullptr, 0, ACT_NONE, 0, &x, y);
        if (tape) tape->res[i][1] = raw;
        x = y;
    }
    if (tape) tape->op_up[0] = x;
    x = conv_in_relu(up_[0], up_n_[0], x, b * 2, nullptr, tape ? &tape->up[0] : nullptr);
    if (tape) tape->op_up[1] = x;
    x = conv_in_relu(up_[1], up_n_[1], x, b * 4, nullptr, tape ? &tape->up[1] : nullptr);
    if (tape) tape->op_up[2] = x;
    // last block: leave InstanceNorm + ReLU pending; the tail kernel applies them while staging its halo tile
    View raw = make_view(P, B, S_, S_, 64, &rt);
    run_conv(rt, up_[2], x, raw);
    if (tape) tape->up[2] = raw;
    float* coef = tail_coef(rt, raw, up_n_[2], 0);
    tail_forward(kind_, tail_, raw, coef, ACT_RELU, image0, image1, outputs, s, rt.strict);
}

// Default mode (poser_encoder_decoder_00.py:99-121 / face_morpher_08.py:158-168): every InstanceNorm + ReLU between two
// convs is applied by the CONSUMER conv to its operand tiles (ConvNormIn); raw conv outputs live in f16.  What remains as
// a pass: the bottleneck entry (its result is both a residual stream and an operand) and the end of each ResnetBlock
// (x + IN(conv(...)), resnet_block.py:64-67).
void EncDecNet::forward_fused(Runtime& rt, const View& x0, const ImgView& image0, const ImgView& image1, const float* pose,
                              int pose_ld, float* const* outputs, EncDecTape* tape) {
    const int B = x0.N;
    cudaStream_t s = rt.stream;
    Pool* P = rt.persist;
    Tens r0 = make_act(P, rt, B, S_, S_, 64, false, true);
    run_conv_tc(rt, down_[0], x0, nullptr, r0);                                  // fp32 image operand (kind::tf32)
    if (tape) { tape->down[0] = raw_view(r0); tape->op_down[0] = x0; }
    Tens prev = r0;
    for (int i = 1; i < 3; ++i) {
        Tens r = make_act(P, rt, B, S_ >> i, S_ >> i, down_[i].cout, false, true);
        const ConvNormIn ni = norm_in(prev.f, down_n_[i - 1], 0, ACT_RELU);
        run_conv_tc(rt, down_[i], prev.h, &ni, r);
        if (tape) { tape->down[i] = raw_view(r); tape->op_down[i] = prev.h; }
        prev = r;
    }
    const int b = S_ / 8;
    View bin16 = make_view16(P, B, b, b, 512 + pose_pad_);
    Tens r3 = make_act(P, rt, B, b, b, 512, false, false);                        // statistics slot; the data goes into bin16[:, 0:512]
    r3.h = bin16.slice(0, 512);
    {
        const ConvNormIn ni = norm_in(prev.f, down_n_[2], 0, ACT_RELU);
        run_conv_tc(rt, down_[3], prev.h, &ni, r3);
        if (tape) { tape->down[3] = raw_view(r3); tape->op_down[3] = prev.h; }
    }
    if (pose_pad_ > 0) tile_vector(pose, pose_ld, pose_ch_, bin16.slice(512, pose_pad_), s);   // poser_encoder_decoder_00.py:110-113
    // bottleneck entry: conv -> IN -> ReLU; the result x is a residual stream (fp32) and a conv operand (f16 copy)
    View x = make_view(P, B, b, b, bott0_.cout, &rt);
    View x16 = make_view16(P, B, b, b, bott0_.cout);
    {
        Tens xr; xr.f = x;
        const ConvNormIn ni = norm_in(r3.f, down_n_[3], 0, ACT_RELU, nullptr, nullptr, 0, 512);
        run_conv_tc(rt, bott0_, bin16, &ni, xr);
        if (tape) tape->op_bott0 = bin16;
        const View y = tape ? make_view(P, B, b, b, bott0_.cout) : x;
        run_norm(rt, x, bott0_n_, 0, nullptr, nullptr, 0, ACT_RELU, 0, nullptr, y, &x16);
        if (tape) tape->bott0 = x;
        x = y;
    }
    for (int i = 0; i < 5; ++i) {   // ResnetBlock: x + IN(conv(relu(IN(conv(x)))))  (resnet_block.py:52-67)
        Tens ha = make_act(P, rt, B, b, b, 512, false, true);
        run_conv_tc(rt, res_[i][0], x16, nullptr, ha);
        Tens hb = make_act(P, rt, B, b, b, 512, true, false);
        const ConvNormIn ni = norm_in(ha.f, res_n_[i][0], 0, ACT_RELU);
        run_conv_tc(rt, res_[i][1], ha.h, &ni, hb);
        View n16 = make_view16(P, B, b, b, 512);
        const View y = tape ? make_view(P, B, b, b, 512) : hb.f;
        run_norm(rt, hb.f, res_n_[i][1], 0, nullptr, nullptr, 0, ACT_NONE, 0, &x, y, &n16);
        if (tape) { tape->res[i][0] = raw_view(ha); tape->res[i][1] = hb.f; tape->op_res[i][0] = x16; tape->op_res[i][1] = ha.h; }
        x = y; x16 = n16;
    }
    Tens u0 = make_act(P, rt, B, 2 * b, 2 * b, up_[0].cout, false, true);
    run_conv_tc(rt, up_[0], x16, nullptr, u0);
    Tens u1 = make_act(P, rt, B, 4 * b, 4 * b, up_[1].cout, false, true);
    {
        const ConvNormIn ni = norm_in(u0.f, up_n_[0], 0, ACT_RELU);
        run_conv_tc(rt, up_[1], u0.h, &ni, u1);
    }
    if (tape) { tape->up[0] = raw_view(u0); tape->up[1] = raw_view(u1); tape->op_up[0] = x16; tape->op_up[1] = u0.h; tape->op_up[2] = u1.h; }
    // last block: InstanceNorm + ReLU stay pending; the tail kernel applies them while staging its halo tile
    const bool tc_tail = tail_.w16 != nullptr;
    Tens feat = make_act(P, rt, B, S_, S_, 64, !tc_tail, tc_tail);
    {
        const ConvNormIn ni = norm_in(u1.f, up_n_[1], 0, ACT_RELU);
        run_conv_tc(rt, up_[2], u1.h, &ni, feat);
    }
    if (tape) tape->up[2] = raw_view(feat);
    if (tc_tail) {
        const View fv = with_stats(feat.h, feat.f);       // f16 data + the statistics slot of the tensor
        NormSpecTail ns; ns.groups = 0; ns.act = ACT_RELU; ns.gamma = up_n_[2].gamma; ns.beta = up_n_[2].beta;
        // the network's own NHWC input holds interleaved copies of the image(s) the tail samples (combiner: [background | eyebrow])
        const View g0 = kind_ == TAIL_COMBINER ? x0.slice(4, 4) : x0.slice(0, 4);
        const View g1 = x0.slice(0, 4);
        tail_tc_forward(kind_, tail_, fv, ns, image0, image1, outputs, s, &g0, kind_ == TAIL_COMBINER ? &g1 : nullptr);
    } else {
        float* coef = tail_coef(rt, feat.f, up_n_[2], 0);
        tail_forward(kind_, tail_, feat.f, coef, ACT_RELU, image0, image1, outputs, s, rt.strict);
    }
}

// ------------------------------------------------------------------------------------------------ UNetNet
UNetNet::UNetNet(bool upscaler, int size, int model_channels, std::vector<int> mults)
    : upscaler_(upscaler), S_(size), mc_(model_channels), L_((int)mults.size()), mults_(std::move(mults)), cat_h_(2 * L_),
      cat_skip_(2 * L_) {
    // the skip tensors hs[k] in down-path order: the first conv's output, then per level its ResBlock's and (but on the last
    // level) its down-sampler's
    std::vector<int> hs_ch(2 * L_);
    hs_ch[0] = mc_;
    for (int i = 0; i < L_; ++i) {
        hs_ch[2 * i + 1] = mc_ * mults_[i];
        if (i < L_ - 1) hs_ch[2 * i + 2] = mc_ * mults_[i];
    }
    for (int j = 0; j < 2 * L_; ++j) {
        const int lvl = L_ - 1 - j / 2;
        cat_h_[j] = (j == 0) ? mc_ * mults_[L_ - 1] : ((j & 1) ? mc_ * mults_[lvl] : mc_ * mults_[lvl + 1]);
        cat_skip_[j] = hs_ch[2 * L_ - 1 - j];
    }
}

namespace {

ResBlockW load_res_block(const StateDict& sd, const std::string& p, cudaStream_t s, bool upsampling = false) {
    ResBlockW w;
    w.key = p;
    w.norm0 = load_norm(sd, p + ".norm0", s);
    w.conv0 = load_conv(sd, p + ".conv0", upsampling ? CONV_UP2_3x3 : CONV_3x3, true, s);
    w.norm1 = load_norm(sd, p + ".norm1", s);
    w.conv1 = load_conv(sd, p + ".conv1", CONV_3x3, true, s);
    w.cin = w.conv0.cin; w.cout = w.conv0.cout;
    w.has_skip = sd.count(p + ".skip.weight") > 0;
    if (w.has_skip) w.skip = load_conv(sd, p + ".skip", CONV_1x1, true, s);
    // default mode (f16 copies): conv1 and the skip as one K, with bias b1 + b_skip (the separate convs stay: strict mode
    // and the backward's adjoints)
    if (w.has_skip && w.conv1.w16 && w.skip.w16) conv_make_fold(w.fold, w.conv1, w.skip, s);
    return w;
}

AttnW load_attn(const StateDict& sd, const std::string& p, cudaStream_t s) {
    AttnW a;
    a.key = p;
    a.norm = load_norm(sd, p + ".norm", s);
    a.qkv = load_conv(sd, p + ".qkv", CONV_1x1, true, s);
    a.proj = load_conv(sd, p + ".conv", CONV_1x1, true, s);
    a.C = a.proj.cout;
    return a;
}

}  // namespace

void UNetNet::load(const StateDict& sd, cudaStream_t s) {
    SinkScope own(&owned_);
    const std::string p = "body.";
    std::vector<std::pair<ResBlockW*, std::string>> all_blocks;   // for FiLM batching
    // first conv (Upscaler02: first_conv(rest) + coarse_image_conv(cat(coarse_posed, warped, coarse_grid)) fused
    // into one 16-input-channel conv; upscaler_02.py:79-82, unet.py:645-646)
    if (!upscaler_) {
        first_ = load_conv(sd, p + "first_conv", CONV_3x3, true, s);
    } else {
        const TensorRef& w1 = sd_get(sd, p + "first_conv.weight");
        const TensorRef& w2 = sd_get(sd, "coarse_image_conv.weight");
        THA4_REQUIRE(w1.shape[1] == 4 && w2.shape[1] == 10 && w1.shape[0] == w2.shape[0], "upscaler first conv shapes");
        conv_describe(first_, CONV_3x3, 16, (int)w1.shape[0]);
        first_.w = dev_alloc(conv_packed_floats(first_));
        THA4_CUDA_CHECK(cudaMemsetAsync(first_.w, 0, conv_packed_floats(first_) * sizeof(float), s));
        conv_pack(first_, CONV_3x3, w1.p, 4, 0, s);
        conv_pack(first_, CONV_3x3, w2.p, 10, 4, s);
        first_.tf32_rounded = conv_pack_rounding();
        first_.bias = dev_alloc(first_.cout);
        vec_add_kernel<<<ceil_div(first_.cout, 128), 128, 0, s>>>(first_.bias, sd_get(sd, p + "first_conv.bias").p,
                                                                  sd_get(sd, "coarse_image_conv.bias").p, first_.cout);
        THA4_LAUNCH_CHECK();
    }
    down_res_.resize(L_); down_ds_.resize(L_ - 1);
    for (int i = 0; i < L_; ++i) {
        const std::string bp = p + "down_blocks." + std::to_string(i);
        down_res_[i] = load_res_block(sd, bp + ".res_blocks.0", s);
        all_blocks.push_back({&down_res_[i], bp + ".res_blocks.0"});
        if (i == L_ - 1) down_attn_ = load_attn(sd, bp + ".attention_blocks.0", s);
        if (i < L_ - 1) {
            down_ds_[i] = load_res_block(sd, bp + ".downsample", s);
            all_blocks.push_back({&down_ds_[i], bp + ".downsample"});
        }
    }
    mid_res_.resize(4); mid_attn_.resize(3);
    for (int j = 0; j < 7; ++j) {
        const std::string mp = p + "middle_blocks." + std::to_string(j);
        if (j % 2 == 0) { mid_res_[j / 2] = load_res_block(sd, mp, s); all_blocks.push_back({&mid_res_[j / 2], mp}); }
        else mid_attn_[j / 2] = load_attn(sd, mp + ".module", s);
    }
    up_res_.resize(2 * L_); up_us_.resize(L_ - 1); up_attn_.resize(2);
    for (int bi = 0; bi < L_; ++bi) {
        const std::string bp = p + "up_blocks." + std::to_string(bi);
        for (int r = 0; r < 2; ++r) {
            const std::string rp = bp + ".resnet_blocks." + std::to_string(r);
            up_res_[2 * bi + r] = load_res_block(sd, rp, s);
            all_blocks.push_back({&up_res_[2 * bi + r], rp});
            if (bi == 0) up_attn_[r] = load_attn(sd, bp + ".attention_blocks." + std::to_string(r), s);
        }
        if (bi < L_ - 1) {
            up_us_[bi] = load_res_block(sd, bp + ".upsample", s, true);
            all_blocks.push_back({&up_us_[bi], bp + ".upsample"});
        }
    }
    for (int j = 0; j < 2 * L_; ++j) {
        THA4_REQUIRE(cat_h_[j] + cat_skip_[j] == up_res_[j].cin, "unet: concat plan does not match weights");
        THA4_REQUIRE(up_res_[j].has_skip, "unet: an up ResBlock reads its concatenation through a 1x1 skip (no fp32 residual)");
    }
    last_n_ = load_norm(sd, p + "last.0", s);
    tail_init(tail_, mc_, s);
    tail_add_head(tail_, sd, p + "last.2", true, s);

    // pose embedding MLP (unet.py:449-452)
    cond_w0_ = dev_clone(sd_get(sd, p + "cond_embed.0.weight"), s);
    cond_b0_ = dev_clone(sd_get(sd, p + "cond_embed.0.bias"), s);
    cond_w2_ = dev_clone(sd_get(sd, p + "cond_embed.2.weight"), s);
    cond_b2_ = dev_clone(sd_get(sd, p + "cond_embed.2.bias"), s);

    // time embedding at t = 0 is a constant: cat(cos(0)..., sin(0)...) -> Linear -> SiLU -> Linear  (unet.py:365-376,443-447)
    std::vector<float> t0(mc_, 0.0f);
    for (int i = 0; i < mc_ / 2; ++i) t0[i] = 1.0f;
    // kept (with time_embed.3's weight) for the parameter gradients
    float* d_t0 = dev_alloc(mc_);
    THA4_CUDA_CHECK(cudaMemcpyAsync(d_t0, t0.data(), mc_ * sizeof(float), cudaMemcpyHostToDevice, s));
    float* d_t1 = dev_alloc(256);
    float* d_t2 = dev_alloc(256);
    linear_forward(d_t0, mc_, 1, mc_, sd_get(sd, p + "time_embed.1.weight").p, sd_get(sd, p + "time_embed.1.bias").p, 256, 0, d_t1, 256, s);
    linear_forward(d_t1, 256, 1, 256, sd_get(sd, p + "time_embed.3.weight").p, sd_get(sd, p + "time_embed.3.bias").p, 256, 1, d_t2, 256, s);

    // per-block FiLM: cond0 (time) folded to constants; cond1 (pose) stacked into one [R,256] projection
    film1_total_ = 0;
    for (auto& e : all_blocks) { e.first->film1_off = film1_total_; film1_total_ += 2 * e.first->cout; }
    film1_w_ = dev_alloc((size_t)film1_total_ * 256);
    film1_b_ = dev_alloc(film1_total_);
    film0_w_ = dev_alloc((size_t)film1_total_ * 256);
    for (auto& e : all_blocks) {
        ResBlockW* w = e.first;
        const TensorRef& c0w = sd_get(sd, e.second + ".cond0_layers.1.weight");
        THA4_REQUIRE(c0w.shape[0] == 2 * w->cout && c0w.shape[1] == 256, "cond0 shape: " + e.second);
        w->film0 = dev_alloc(2 * w->cout);
        linear_forward(d_t2, 256, 1, 256, c0w.p, sd_get(sd, e.second + ".cond0_layers.1.bias").p, 2 * w->cout, 1, w->film0, 2 * w->cout, s);
        THA4_CUDA_CHECK(cudaMemcpyAsync(film0_w_ + (size_t)w->film1_off * 256, c0w.p, c0w.numel() * sizeof(float), cudaMemcpyDeviceToDevice, s));
        const TensorRef& c1w = sd_get(sd, e.second + ".cond1_layers.1.weight");
        THA4_REQUIRE(c1w.shape[0] == 2 * w->cout && c1w.shape[1] == 256, "cond1 shape: " + e.second);
        THA4_CUDA_CHECK(cudaMemcpyAsync(film1_w_ + (size_t)w->film1_off * 256, c1w.p, c1w.numel() * sizeof(float), cudaMemcpyDeviceToDevice, s));
        THA4_CUDA_CHECK(cudaMemcpyAsync(film1_b_ + w->film1_off, sd_get(sd, e.second + ".cond1_layers.1.bias").p,
                                        2 * w->cout * sizeof(float), cudaMemcpyDeviceToDevice, s));
    }
    if (conv_pack_rounding()) tail_make_half(tail_, s);       // default mode: the wgmma tail's f16 head weights
    params_ = ParamLayout();
    time_t0_ = d_t0; time_t1_ = d_t1; time_t2_ = d_t2;
    time_w3_ = dev_clone(sd_get(sd, p + "time_embed.3.weight"), s);
    // the flat parameter-gradient layout: the reference's state_dict order (unet.py:438-529, registration order of the
    // modules; per up level its ResBlocks, then its attention blocks, then the up-sampler)
    auto reg_res = [&](const ResBlockW& w) {
        for (const char* k : {".norm0.weight", ".norm0.bias", ".conv0.weight", ".conv0.bias", ".cond0_layers.1.weight",
                              ".cond0_layers.1.bias", ".norm1.weight", ".norm1.bias", ".conv1.weight", ".conv1.bias",
                              ".cond1_layers.1.weight", ".cond1_layers.1.bias"})
            params_.add(sd, w.key + k);
        if (w.has_skip) { params_.add(sd, w.key + ".skip.weight"); params_.add(sd, w.key + ".skip.bias"); }
    };
    auto reg_attn = [&](const AttnW& a) {
        for (const char* k : {".norm.weight", ".norm.bias", ".qkv.weight", ".qkv.bias", ".conv.weight", ".conv.bias"})
            params_.add(sd, a.key + k);
    };
    for (const char* k : {"time_embed.1.weight", "time_embed.1.bias", "time_embed.3.weight", "time_embed.3.bias", "cond_embed.0.weight",
                          "cond_embed.0.bias", "cond_embed.2.weight", "cond_embed.2.bias", "first_conv.weight", "first_conv.bias"})
        params_.add(sd, p + k);
    for (int i = 0; i < L_; ++i) {
        reg_res(down_res_[i]);
        if (i == L_ - 1) reg_attn(down_attn_);
        if (i < L_ - 1) reg_res(down_ds_[i]);
    }
    for (int j = 0; j < 7; ++j) { if (j % 2 == 0) reg_res(mid_res_[j / 2]); else reg_attn(mid_attn_[j / 2]); }
    for (int bi = 0; bi < L_; ++bi) {
        reg_res(up_res_[2 * bi]); reg_res(up_res_[2 * bi + 1]);
        if (bi == 0) { reg_attn(up_attn_[0]); reg_attn(up_attn_[1]); }
        if (bi < L_ - 1) reg_res(up_us_[bi]);
    }
    for (const char* k : {"last.0.weight", "last.0.bias", "last.2.weight", "last.2.bias"}) params_.add(sd, p + k);
    if (upscaler_) {      // Upscaler02's own, after the U-Net's
        params_.add(sd, "coarse_image_conv.weight");
        params_.add(sd, "coarse_image_conv.bias");
    }
    THA4_REQUIRE((long)params_.off.size() == (long)sd.size(), "unet: the state_dict has tensors outside the parameter layout");
    THA4_CUDA_CHECK(cudaStreamSynchronize(s));
    loaded_ = true;
}

void ParamLayout::add(const StateDict& sd, const std::string& key) {
    off[key] = total;
    total += sd_get(sd, key).numel();
}

long ParamLayout::offset(const std::string& key) const {
    auto it = off.find(key);
    THA4_REQUIRE(it != off.end(), "parameter gradients: no tensor " + key);
    return it->second;
}

// ResBlock (unet.py:154-165).  mode: 0 same, 1 up (nearest x2), 2 down (AvgPool2d(2)).
void UNetNet::res_block(Runtime& rt, const ResBlockW& w, const View& x, int mode, const float* film1, const View& out, UNetTape* tape) {
    cudaStream_t s = rt.stream;
    rt.scratch->reset();
    THA4_REQUIRE(x.C == w.cin && out.C == w.cout, "res_block: channels");
    const int B = x.N;
    // norm0 -> SiLU -> (avg-pool) ; the nearest-upsample is folded into conv0's gather
    const int th = (mode == 2) ? x.H / 2 : x.H;
    const bool ops = tape && tape->ops;          // the normalised operands stay for the weight gradients
    Pool* op_pool = ops ? rt.persist : rt.scratch;
    View t0 = make_view(op_pool, B, th, th, w.cin);
    run_norm(rt, x, w.norm0, 32, nullptr, nullptr, 0, rt.strict ? ACT_SILU : ACT_SILU_FAST, mode == 2 ? 1 : 0, nullptr, t0);
    View h = make_view(tape ? rt.persist : rt.scratch, B, out.H, out.W, w.cout, &rt);
    run_conv(rt, w.conv0, t0, h);      // mode 1: conv0 was packed as CONV_UP2_3x3 (upsample folded into 4 phases)
    // norm1 -> FiLM(time) -> FiLM(pose) -> SiLU, folded into one per-(n,c) affine
    const View h2 = tape ? make_view(op_pool, B, out.H, out.W, w.cout) : h;
    if (tape) tape->res[&w] = {x, h, ops ? t0 : View{}, ops ? h2 : View{}};
    run_norm(rt, h, w.norm1, 32, w.film0, film1 + w.film1_off, film1_total_, rt.strict ? ACT_SILU : ACT_SILU_FAST, 0, nullptr, h2);
    if (w.has_skip) {
        THA4_REQUIRE(mode == 0, "res_block: skip conv only on same-resolution blocks");
        View sk = make_view(rt.scratch, B, x.H, x.W, w.cout);
        run_conv(rt, w.skip, x, sk);
        run_conv(rt, w.conv1, h2, out, 0, &sk, RES_SAME);
    } else {
        run_conv(rt, w.conv1, h2, out, 0, &x, mode == 0 ? RES_SAME : (mode == 1 ? RES_UP2 : RES_DOWN2));
    }
}

// AttentionBlock (unet.py:230-239)
void UNetNet::attn_block(Runtime& rt, const AttnW& w, const View& x, const View& out, UNetTape* tape) {
    cudaStream_t s = rt.stream;
    rt.scratch->reset();
    const bool ops = tape && tape->ops;
    Pool* op_pool = ops ? rt.persist : rt.scratch;
    View t = make_view(op_pool, x.N, x.H, x.W, x.C);
    run_norm(rt, x, w.norm, 32, nullptr, nullptr, 0, ACT_NONE, 0, nullptr, t);
    View qkv = make_view(tape ? rt.persist : rt.scratch, x.N, x.H, x.W, 3 * x.C);
    run_conv(rt, w.qkv, t, qkv);
    View a = make_view(op_pool, x.N, x.H, x.W, x.C);
    if (tape) tape->attn[&w] = {x, qkv, ops ? t : View{}, ops ? a : View{}};
    attention_forward(qkv, 8, a, s, !rt.strict);
    run_conv(rt, w.proj, a, out, 0, &x, RES_SAME);
}

void UNetNet::forward(Runtime& rt, const ImgView& image, const float* coarse_posed, const float* coarse_grid, int coarse_size,
                      const float* pose, int pose_ld, float* const* outputs, UNetTape* tape) {
    THA4_REQUIRE(loaded_, "network weights not loaded");
    THA4_REQUIRE(image.H == S_ && image.W == S_ && image.C == 4, "unet: image size");
    if (rt.f16) { forward_fused(rt, image, coarse_posed, coarse_grid, coarse_size, pose, pose_ld, outputs, tape); return; }
    const int B = image.N;
    cudaStream_t s = rt.stream;
    Pool* P = rt.persist;
    rt.scratch->reset();

    // pose embedding and all FiLM vectors of this forward in three tiny launches
    float* c1 = P->alloc((size_t)B * 256);
    float* c2 = P->alloc((size_t)B * 256);
    float* film1 = P->alloc((size_t)B * film1_total_);
    linear_forward(pose, pose_ld, B, 6, cond_w0_, cond_b0_, 256, 0, c1, 256, s);
    linear_forward(c1, 256, B, 256, cond_w2_, cond_b2_, 256, 1, c2, 256, s);
    linear_forward(c2, 256, B, 256, film1_w_, film1_b_, film1_total_, 1, film1, film1_total_, s);
    if (tape) { tape->c1 = c1; tape->c2 = c2; tape->film1 = film1; }

    View x0;
    if (upscaler_) {
        x0 = make_view(P, B, S_, S_, 16);
        upscaler_prologue(image, coarse_posed, coarse_grid, coarse_size, x0, s);
    } else {
        x0 = make_view(P, B, S_, S_, 4);
        nchw_to_nhwc(image, x0, s);
    }
    if (tape) tape->x0 = x0;

    // ---- the skip concatenations: up res-block j reads cat(h_j, hs[2L-1-j]) from one buffer ----
    const int NH = 2 * L_;
    std::vector<View> cat(NH), hs(NH);
    for (int j = 0; j < NH; ++j) {
        const int sp = S_ >> (L_ - 1 - j / 2);
        cat[j] = make_view(P, B, sp, sp, cat_h_[j] + cat_skip_[j], &rt);
        hs[NH - 1 - j] = cat[j].slice(cat_h_[j], cat_skip_[j]);
    }

    // ---- down path (unet.py:534-536) ----
    run_conv(rt, first_, x0, hs[0]);
    View cur = hs[0];
    for (int i = 0; i < L_; ++i) {
        if (i == L_ - 1) {
            View tmp = make_view(P, B, cur.H, cur.W, down_res_[i].cout, &rt);
            res_block(rt, down_res_[i], cur, 0, film1, tmp, tape);
            attn_block(rt, down_attn_, tmp, hs[2 * i + 1], tape);
        } else {
            res_block(rt, down_res_[i], cur, 0, film1, hs[2 * i + 1], tape);
        }
        cur = hs[2 * i + 1];
        if (i < L_ - 1) {
            res_block(rt, down_ds_[i], cur, 2, film1, hs[2 * i + 2], tape);
            cur = hs[2 * i + 2];
        }
    }
    // ---- middle: Res, Attn, Res, Attn, Res, Attn, Res (unet.py:481-498) ----
    for (int j = 0; j < 4; ++j) {
        const bool last = (j == 3);
        View r = last ? cat[0].slice(0, cat_h_[0]) : make_view(P, B, cur.H, cur.W, cur.C, &rt);
        res_block(rt, mid_res_[j], cur, 0, film1, r, tape);
        cur = r;
        if (!last) {
            View a = make_view(P, B, cur.H, cur.W, cur.C, &rt);
            attn_block(rt, mid_attn_[j], cur, a, tape);
            cur = a;
        }
    }
    // ---- up path (unet.py:540-544) ----
    View feat;
    for (int j = 0; j < NH; ++j) {
        const int lvl = L_ - 1 - j / 2;
        const bool second = (j & 1);
        const int co = up_res_[j].cout;
        View dst;
        if (!second) dst = cat[j + 1].slice(0, cat_h_[j + 1]);
        else dst = make_view(P, B, cat[j].H, cat[j].W, co, &rt);      // goes to the upsampler or is the final feature
        if (lvl == L_ - 1) {
            View tmp = make_view(P, B, cat[j].H, cat[j].W, co, &rt);
            res_block(rt, up_res_[j], cat[j], 0, film1, tmp, tape);
            attn_block(rt, up_attn_[second ? 1 : 0], tmp, dst, tape);
        } else {
            res_block(rt, up_res_[j], cat[j], 0, film1, dst, tape);
        }
        if (second) {
            if (lvl > 0) res_block(rt, up_us_[L_ - 1 - lvl], dst, 1, film1, cat[j + 1].slice(0, cat_h_[j + 1]), tape);
            else feat = dst;
        }
    }
    // ---- last: GroupNorm + SiLU pending, applied inside the fused tail (unet.py:526-529; morpher_00.py:53-58) ----
    rt.scratch->reset();
    if (tape) tape->feat = feat;
    float* coef = tail_coef(rt, feat, last_n_, 32);
    ImgView none{};
    tail_forward(TAIL_UNET, tail_, feat, coef, rt.strict ? ACT_SILU : ACT_SILU_FAST, image, none, outputs, s, rt.strict);
}

// ------------------------------------------------------------------------------------------------ UNetNet, default mode
// Every GroupNorm (+FiLM) + SiLU that sits between two convs is applied by the consumer conv to its operand tiles
// (ConvNormIn); block outputs (the residual streams) are written once in fp32 and once in f16 by the producing conv.
// Only the down-sampling blocks keep a normalisation pass (SiLU must precede the 2x2 mean, unet.py:58,158).
namespace {

// a normalisation's input as the fused consumer conv reads it: the f16 operand copy when there is one, with the statistics
View op_view(const Tens& a) { return a.h.p ? with_stats(a.h, a.f) : a.f; }

struct UNetFused {
    Runtime& rt;
    const float* film1;
    int film1_total;
    UNetTape* tape;

    // ResBlock (unet.py:154-165).  mode: 0 same, 1 up (nearest x2), 2 down (AvgPool2d(2)).
    void res_block(const ResBlockW& w, const Tens& x, int mode, const Tens& out) {
        rt.scratch->reset();
        // x's fp32 data feeds the down-sampling norm pass or the residual (a block with a 1x1 skip adds skip(x) instead);
        // its f16 copy feeds conv0 (mode 0, 1) and the skip conv
        const bool reads_f32 = mode == 2 || !w.has_skip, reads_f16 = mode != 2 || w.has_skip;
        THA4_REQUIRE(x.f.C == w.cin && out.f.C == w.cout && (x.f.p || !reads_f32) && (x.h.p || !reads_f16),
                     "res_block: the input lacks a precision the block reads");
        const int B = x.f.N;
        const int act = ACT_SILU_FAST;
        Tens h0 = make_act(tape ? rt.persist : rt.scratch, rt, B, out.f.H, out.f.W, w.cout, false, true);
        if (tape) tape->res[&w] = {mode == 2 ? x.f : op_view(x), raw_view(h0)};
        // conv1 with the skip folded into its K loop: one launch, no skip(x) tensor, no fork / join around it
        ConvArgs fa;
        fa.in = h0.h; fa.out = out.f; fa.out16 = out.h; fa.in2 = x.h; fa.nin.on = true;
        const bool fold = mode == 0 && w.fold.cin2 > 0 && opts().skip_fold && conv_halo_supported(w.fold, fa);
        Tens sk;
        if (w.has_skip && !fold) {
            // skip(x) depends on x only: it runs on the side stream next to norm0 -> conv0 (a latency-bound chain,
            // ~30 times per frame) and is joined in front of conv1, which adds it as the residual
            sk = make_act(rt.scratch, rt, B, x.f.H, x.f.W, w.cout, true, false, false);
            if (rt.side) {
                THA4_CUDA_CHECK(cudaEventRecord(rt.ev_fork, rt.stream));
                THA4_CUDA_CHECK(cudaStreamWaitEvent(rt.side, rt.ev_fork, 0));
                cudaStream_t main_stream = rt.stream;
                rt.stream = rt.side;
                try { run_conv_tc(rt, w.skip, x.h, nullptr, sk); } catch (...) { rt.stream = main_stream; throw; }
                rt.stream = main_stream;
                THA4_CUDA_CHECK(cudaEventRecord(rt.ev_join, rt.side));
            } else {
                run_conv_tc(rt, w.skip, x.h, nullptr, sk);
            }
        }
        View xpool;
        if (mode == 2) {          // norm0 -> SiLU -> 2x2 mean as a pass (f16 result), then a plain conv
            View t0 = make_view16(tape && tape->ops ? rt.persist : rt.scratch, B, x.f.H / 2, x.f.W / 2, w.cin);
            if (tape && tape->ops) tape->res[&w].t0 = t0;
            xpool = make_view(rt.scratch, B, x.f.H / 2, x.f.W / 2, w.cin);       // AvgPool2d(2) of the skip path, written by the same pass
            run_norm(rt, x.f, w.norm0, 32, nullptr, nullptr, 0, act, 1, nullptr, t0, nullptr, &xpool);
            run_conv_tc(rt, w.conv0, t0, nullptr, h0);
        } else {                  // mode 1: conv0 was packed as CONV_UP2_3x3 (the upsample is folded into 4 phases of the low-res input)
            const ConvNormIn n0 = norm_in(x.f, w.norm0, 32, act);
            run_conv_tc(rt, w.conv0, x.h, &n0, h0);
        }
        // norm1 -> FiLM(time) -> FiLM(pose) -> SiLU, folded into one per-(n,c) affine inside conv1
        const ConvNormIn n1 = norm_in(h0.f, w.norm1, 32, act, w.film0, film1 + w.film1_off, film1_total);
        if (fold) {
            run_conv_tc(rt, w.fold, h0.h, &n1, out, nullptr, RES_NONE, &x.h);
        } else if (w.has_skip) {
            THA4_REQUIRE(mode == 0, "res_block: skip conv only on same-resolution blocks");
            if (rt.side) THA4_CUDA_CHECK(cudaStreamWaitEvent(rt.stream, rt.ev_join, 0));
            run_conv_tc(rt, w.conv1, h0.h, &n1, out, &sk.f, RES_SAME);
        } else {
            if (mode == 2) run_conv_tc(rt, w.conv1, h0.h, &n1, out, &xpool, RES_SAME);
            else run_conv_tc(rt, w.conv1, h0.h, &n1, out, &x.f, mode == 0 ? RES_SAME : RES_UP2);
        }
    }

    // AttentionBlock (unet.py:230-239): GroupNorm fused into the qkv conv
    void attn_block(const AttnW& w, const Tens& x, const Tens& out) {
        rt.scratch->reset();
        Tens qkv = make_act(tape ? rt.persist : rt.scratch, rt, x.f.N, x.f.H, x.f.W, 3 * x.f.C, true, false, false);
        const ConvNormIn n = norm_in(x.f, w.norm, 32, ACT_NONE);
        run_conv_tc(rt, w.qkv, x.h, &n, qkv);
        View a = make_view(tape && tape->ops ? rt.persist : rt.scratch, x.f.N, x.f.H, x.f.W, x.f.C);
        if (tape) tape->attn[&w] = {op_view(x), qkv.f, View{}, tape->ops ? a : View{}};
        attention_forward(qkv.f, 8, a, rt.stream, true);
        run_conv_tc(rt, w.proj, a, nullptr, out, &x.f, RES_SAME);
    }
};

}  // namespace

void UNetNet::forward_fused(Runtime& rt, const ImgView& image, const float* coarse_posed, const float* coarse_grid, int coarse_size,
                            const float* pose, int pose_ld, float* const* outputs, UNetTape* tape) {
    const int B = image.N;
    cudaStream_t s = rt.stream;
    Pool* P = rt.persist;
    rt.scratch->reset();

    float* c1 = P->alloc((size_t)B * 256);
    float* c2 = P->alloc((size_t)B * 256);
    float* film1 = P->alloc((size_t)B * film1_total_);
    // the pose MLP + FiLM projection (three dependent GEMVs, ~25 us) is first needed by conv1 of the first ResBlock: it runs on
    // the side stream next to the prologue, the first conv and conv0
    cudaStream_t ls = s;
    if (rt.side) {
        THA4_CUDA_CHECK(cudaEventRecord(rt.ev_fork, s));
        THA4_CUDA_CHECK(cudaStreamWaitEvent(rt.side, rt.ev_fork, 0));
        ls = rt.side;
    }
    linear_forward(pose, pose_ld, B, 6, cond_w0_, cond_b0_, 256, 0, c1, 256, ls);
    linear_forward(c1, 256, B, 256, cond_w2_, cond_b2_, 256, 1, c2, 256, ls);
    linear_forward(c2, 256, B, 256, film1_w_, film1_b_, film1_total_, 1, film1, film1_total_, ls);
    if (rt.side) THA4_CUDA_CHECK(cudaEventRecord(rt.ev_join, rt.side));
    if (tape) { tape->c1 = c1; tape->c2 = c2; tape->film1 = film1; }
    UNetFused F{rt, film1, film1_total_, tape};

    View x0;
    if (upscaler_) {
        x0 = make_view(P, B, S_, S_, 16);
        upscaler_prologue(image, coarse_posed, coarse_grid, coarse_size, x0, s);
    } else {
        x0 = make_view(P, B, S_, S_, 4);
        nchw_to_nhwc(image, x0, s);
    }
    if (tape) tape->x0 = x0;

    // ---- the skip concatenations: up res-block j reads cat(h_j, hs[2L-1-j]) from one buffer (both precisions) ----
    const int NH = 2 * L_;
    std::vector<Tens> cat(NH), hs(NH);
    for (int j = 0; j < NH; ++j) {
        const int sp = S_ >> (L_ - 1 - j / 2);
        cat[j] = make_act(P, rt, B, sp, sp, cat_h_[j] + cat_skip_[j], true, true);
        hs[NH - 1 - j] = slice_act(cat[j], cat_h_[j], cat_skip_[j]);
    }

    // ---- down path (unet.py:534-536) ----
    run_conv_tc(rt, first_, x0, nullptr, hs[0]);
    if (rt.side) THA4_CUDA_CHECK(cudaStreamWaitEvent(s, rt.ev_join, 0));        // FiLM table ready
    Tens cur = hs[0];
    for (int i = 0; i < L_; ++i) {
        if (i == L_ - 1) {
            Tens tmp = make_act(P, rt, B, cur.f.H, cur.f.W, down_res_[i].cout, true, true);
            F.res_block(down_res_[i], cur, 0, tmp);
            F.attn_block(down_attn_, tmp, hs[2 * i + 1]);
        } else {
            F.res_block(down_res_[i], cur, 0, hs[2 * i + 1]);
        }
        cur = hs[2 * i + 1];
        if (i < L_ - 1) {
            // read by the next ResBlock and, through cat, by an up ResBlock: in fp32 only as the former's residual
            cur = down_res_[i + 1].has_skip ? f16_only(hs[2 * i + 2]) : hs[2 * i + 2];
            F.res_block(down_ds_[i], hs[2 * i + 1], 2, cur);
        }
    }
    // ---- middle: Res, Attn, Res, Attn, Res, Attn, Res (unet.py:481-498) ----
    for (int j = 0; j < 4; ++j) {
        const bool last = (j == 3);
        Tens r = last ? f16_only(slice_act(cat[0], 0, cat_h_[0])) : make_act(P, rt, B, cur.f.H, cur.f.W, cur.f.C, true, true);
        F.res_block(mid_res_[j], cur, 0, r);
        cur = r;
        if (!last) {
            Tens a = make_act(P, rt, B, cur.f.H, cur.f.W, cur.f.C, true, true);
            F.attn_block(mid_attn_[j], cur, a);
            cur = a;
        }
    }
    // ---- up path (unet.py:540-544) ----
    // The up half of cat[j] is read by up ResBlock j only, which has a 1x1 skip (cin = both halves): f16 and statistics.
    // The second block of a level feeds the up-sampler (fp32 residual) or, at the top, the tail (f16 on the wgmma tail).
    const bool tc_tail = tail_.w16 != nullptr;
    Tens feat;
    for (int j = 0; j < NH; ++j) {
        const int lvl = L_ - 1 - j / 2;
        const bool second = (j & 1);
        const int co = up_res_[j].cout;
        Tens dst;
        if (!second) dst = f16_only(slice_act(cat[j + 1], 0, cat_h_[j + 1]));
        else dst = make_act(P, rt, B, cat[j].f.H, cat[j].f.W, co, lvl > 0 || !tc_tail, true);   // goes to the upsampler or is the final feature
        if (lvl == L_ - 1) {
            Tens tmp = make_act(P, rt, B, cat[j].f.H, cat[j].f.W, co, true, true);
            F.res_block(up_res_[j], cat[j], 0, tmp);
            F.attn_block(up_attn_[second ? 1 : 0], tmp, dst);
        } else {
            F.res_block(up_res_[j], cat[j], 0, dst);
        }
        if (second) {
            if (lvl > 0) F.res_block(up_us_[L_ - 1 - lvl], dst, 1, f16_only(slice_act(cat[j + 1], 0, cat_h_[j + 1])));
            else feat = dst;
        }
    }
    // ---- last: GroupNorm + SiLU pending, applied inside the fused tail (unet.py:526-529; morpher_00.py:53-58) ----
    rt.scratch->reset();
    ImgView none{};
    if (tc_tail) {
        const View fv = with_stats(feat.h, feat.f);
        NormSpecTail ns; ns.groups = 32; ns.act = ACT_SILU_FAST; ns.gamma = last_n_.gamma; ns.beta = last_n_.beta;
        if (tape) tape->feat = fv;
        const View g0 = x0.slice(0, 4);       // channels 0-3 of the network input are the image the tail warps (Upscaler02: the rest image)
        tail_tc_forward(TAIL_UNET, tail_, fv, ns, image, none, outputs, s, &g0);
    } else {
        if (tape) tape->feat = feat.f;
        float* coef = tail_coef(rt, feat.f, last_n_, 32);
        tail_forward(TAIL_UNET, tail_, feat.f, coef, ACT_SILU_FAST, image, none, outputs, s, rt.strict);
    }
}

}  // namespace tha4
