// extern "C" boundary of libtha4_b200.so (see include/tha4_b200.h) and the poser-level pipelines.
#include "../../include/tha4_b200.h"
#include "nets.cuh"
#include "siren.cuh"
#include "profiler.cuh"
#include "distill.cuh"
#include <atomic>
#include <cstring>
#include <map>
#include <tuple>
#include <vector>

namespace tha4 {
std::atomic<long> g_kernel_launches{0};
bool g_use_pdl = true;
thread_local AllocSink* g_alloc_sink = nullptr;
void* tracked_malloc(size_t bytes) {
    void* p = nullptr;
    THA4_CUDA_CHECK(cudaMalloc(&p, std::max<size_t>(bytes, 16)));
    if (g_alloc_sink) g_alloc_sink->ptrs.push_back(p);
    return p;
}
}

using namespace tha4;

// A whole single-chunk teacher forward captured as a CUDA graph, ZERO-COPY: the graph is captured on the caller's own
// buffers and keyed by their addresses (image, pose, every output, the cached decomposer tensors).  In a steady loop
// -- an app posing into the same tensors, PyTorch's caching allocator handing back the same blocks -- the key repeats and
// the ~260 launches of a frame become one cudaGraphLaunch; a key seen for the second time is captured, at most
// GRAPH_CACHE graphs are kept (least recently used is dropped), and a context whose keys never repeat stops trying.
struct TeacherGraph {
    cudaGraphExec_t exec = nullptr;
    size_t stats_end = 0;      // statistics-arena doubles the pass leaves dirty
    long launches = 0;         // kernels per replay (for the launch counter)
    long last_use = 0;
};
constexpr int GRAPH_CACHE = 8;

struct tha4_ctx {
    int device = 0;
    int use_graphs = 1;        // option "cuda_graphs" (default on): single-chunk teacher forwards replay as one graph launch
    std::map<std::vector<uintptr_t>, TeacherGraph> graphs;
    std::map<std::vector<uintptr_t>, int> graph_seen;      // how often a key was seen before it was captured
    long graph_clock = 0, graph_misses = 0, graph_pause = 0, graph_replays = 0, graph_captures = 0, graph_failures = 0;
    int side_streams = 1;        // option "side_stream": independent DAG branches (ResBlock skip convs) on a second stream
    cudaStream_t side = nullptr;
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
    cudaStream_t capture_stream = nullptr;   // the legacy default stream cannot be captured: its graphs are recorded here and launched there
    float* pose_stage = nullptr;   // [1024][45]: graphs read the pose from here, so the caller's pose address is not part of the key
    void drop_graphs() {
        for (auto& kv : graphs)
            if (kv.second.exec) cudaGraphExecDestroy(kv.second.exec);
        graphs.clear();
        graph_seen.clear();
        graph_misses = 0;
        graph_pause = 0;
    }
    std::string err;
    int strict = 0;
    int microbatch = 32;                   // frames per internal pass
    int half_operands = 1;                 // f16 conv operands between normalisation and wgmma conv (non-strict mode)
    Pool persist, scratch;
    int* flag = nullptr;
    double* loss_acc = nullptr;            // 4 doubles: L1 sums of the distillation step
    double* stats_base = nullptr;          // zero-initialised statistics arena (Runtime::alloc_stats)
    size_t stats_cap = 0, stats_off = 0;
    std::unique_ptr<EncDecNet> decomposer, combiner, face;
    std::unique_ptr<UNetNet> body, upscaler;
    std::unique_ptr<SirenFaceNet> sface;
    std::unique_ptr<SirenBodyNet> sbody;
};

namespace {

thread_local std::string g_create_err;

template <typename F>
int guarded(tha4_ctx* ctx, F&& f) {
    if (!ctx) return THA4_ERR_INVALID;
    try {
        THA4_CUDA_CHECK(cudaSetDevice(ctx->device));
        f();
        return THA4_OK;
    } catch (const CudaError& e) {
        ctx->err = e.what();
        return THA4_ERR_CUDA;
    } catch (const std::exception& e) {
        ctx->err = e.what();
        return THA4_ERR_INVALID;
    }
}

Runtime make_rt(tha4_ctx* ctx, void* stream) {
    Runtime rt;
    rt.persist = &ctx->persist; rt.scratch = &ctx->scratch; rt.stream = (cudaStream_t)stream; rt.strict = ctx->strict;
    rt.f16 = ctx->half_operands && !ctx->strict && conv_tc_enabled();
    rt.stats_base = ctx->stats_base; rt.stats_cap = ctx->stats_cap; rt.stats_off = &ctx->stats_off;
    if (ctx->side_streams && !prof_enabled()) {
        if (!ctx->side) {
            THA4_CUDA_CHECK(cudaStreamCreateWithFlags(&ctx->side, cudaStreamNonBlocking));
            THA4_CUDA_CHECK(cudaEventCreateWithFlags(&ctx->ev_fork, cudaEventDisableTiming));
            THA4_CUDA_CHECK(cudaEventCreateWithFlags(&ctx->ev_join, cudaEventDisableTiming));
        }
        rt.side = ctx->side; rt.ev_fork = ctx->ev_fork; rt.ev_join = ctx->ev_join;
    }
    return rt;
}

// one micro-batch of the teacher pipeline (mode_07.py:72-132 / mode_12.py:66-94)
void teacher_chunk(tha4_ctx* ctx, Runtime& rt, int mode, const float* image, long image_sn, const float* pose, int b, float* const* out,
                   int eyebrow_index, const float* const* cached) {
    cudaStream_t s = rt.stream;
    const int base = (mode == 7) ? 11 : 0;          // index of face_morpher outputs
    float* const* o_face = out + base;
    float* const* o_comb = out + base + 8;
    float* const* o_dec = out + base + 16;
    ImgView img = make_img(image, b, 4, 512, 512);
    img.sn = image_sn;                               // 0: one image posed b times (pose sweep), no replicated copies
    THA4_REQUIRE(eyebrow_index >= 0 && eyebrow_index < 8 && eyebrow_index != 1 && eyebrow_index != 4 && eyebrow_index != 7,
                 "eyebrow_morphed_image_index must select a 4-channel combiner output");
    const float* dec[6];
    if (cached) {
        for (int i = 0; i < 6; ++i) dec[i] = cached[i];
    } else {
        ctx->decomposer->forward(rt, crop_img(img, 64, 192, 128, 128), ImgView{}, nullptr, 0, o_dec);   // mode_07.py:74
        for (int i = 0; i < 6; ++i) dec[i] = o_dec[i];
    }
    // combiner(background_layer = dec[3], eyebrow_layer = dec[0], pose[:, :12])   (mode_07.py:76-84)
    ctx->combiner->forward(rt, make_img(dec[0], b, 4, 128, 128), make_img(dec[3], b, 4, 128, 128), pose, 45, o_comb);
    // face morpher input: 192x192 crop with the morphed eyebrows pasted in   (mode_07.py:89-91)
    float* face_in = ctx->persist.alloc((size_t)b * 4 * 192 * 192);
    copy_window(crop_img(img, 32, 160, 192, 192), face_in, 4L * 192 * 192, 192L * 192, 192, s);
    copy_window(make_img(o_comb[eyebrow_index], b, 4, 128, 128), face_in + 32 * 192 + 32, 4L * 192 * 192, 192L * 192, 192, s);
    ctx->face->forward(rt, make_img(face_in, b, 4, 192, 192), ImgView{}, pose + 12, 45, o_face);
    if (mode != 7) return;
    // face_morphed_full (mode_07.py:93-98) and face_morphed_half (:99-103)
    float* full = out[5];
    copy_window(img, full, 4L * 512 * 512, 512L * 512, 512, s);
    copy_window(make_img(o_face[0], b, 4, 192, 192), full + 32 * 512 + 160, 4L * 512 * 512, 512L * 512, 512, s);
    const ImgView fullv = make_img(full, b, 4, 512, 512);
    float* half = ctx->persist.alloc((size_t)b * 4 * 256 * 256);
    resize_bilinear(fullv, half, 256, 256, s);
    ctx->body->forward(rt, make_img(half, b, 4, 256, 256), nullptr, nullptr, 0, pose + 39, 45, out + 6);
    ctx->upscaler->forward(rt, fullv, out[6], out[9], 256, pose + 39, 45, out + 0);
}

struct OutSpec { int c, s; };
const OutSpec kEncDecDecomposer[6] = {{4, 128}, {1, 128}, {4, 128}, {4, 128}, {1, 128}, {4, 128}};
const OutSpec kCombiner[8] = {{4, 128}, {1, 128}, {4, 128}, {4, 128}, {1, 128}, {4, 128}, {4, 128}, {2, 128}};
const OutSpec kFace[8] = {{4, 192}, {1, 192}, {4, 192}, {4, 192}, {1, 192}, {4, 192}, {4, 192}, {2, 192}};
const OutSpec kSirenBody[5] = {{4, 512}, {1, 512}, {4, 512}, {4, 512}, {2, 512}};

void fill_unet_spec(OutSpec* o, int S) { o[0] = {4, S}; o[1] = {1, S}; o[2] = {4, S}; o[3] = {2, S}; o[4] = {4, S}; }

StateDict make_sd(int n, const char* const* keys, const void* const* ptrs, const int64_t* shapes, const int* ndims) {
    StateDict sd;
    for (int i = 0; i < n; ++i) {
        TensorRef t;
        t.p = reinterpret_cast<const float*>(ptrs[i]);
        for (int d = 0; d < ndims[i]; ++d) t.shape.push_back((long)shapes[4 * i + d]);
        sd[keys[i]] = t;
    }
    return sd;
}

// Start of one pass over the workspace: every pool block becomes reusable and the part of the statistics arena the
// previous pass dirtied is re-zeroed (the arena is all-zero at the start of every pass).
void begin_pass(tha4_ctx* ctx, cudaStream_t stream) {
    ctx->persist.reset();
    ctx->scratch.reset();
    if (ctx->stats_off > 0) THA4_CUDA_CHECK(cudaMemsetAsync(ctx->stats_base, 0, ctx->stats_off * sizeof(double), stream));
    ctx->stats_off = 0;
}

// Runs `fn(chunk offset n0, chunk size b)` over micro-batches of at most `chunk` frames; resets the workspace per chunk.
template <typename F>
void for_chunks(tha4_ctx* ctx, int B, int chunk, cudaStream_t stream, F&& fn) {
    THA4_REQUIRE(B >= 1, "batch must be >= 1");
    for (int n0 = 0; n0 < B; n0 += chunk) {
        const int b = std::min(chunk, B - n0);
        begin_pass(ctx, stream);
        fn(n0, b);
    }
}

template <int NOUT>
void offset_outputs(float* const* outputs, const OutSpec* spec, int n0, float** dst) {
    for (int i = 0; i < NOUT; ++i) dst[i] = outputs[i] + (size_t)n0 * spec[i].c * spec[i].s * spec[i].s;
}

// the upstream gradients of one micro-batch (an entry may be null)
template <int NOUT>
void offset_grads(const float* const* grads, const OutSpec* spec, int n0, const float** dst) {
    for (int i = 0; i < NOUT; ++i) dst[i] = (grads && grads[i]) ? grads[i] + (size_t)n0 * spec[i].c * spec[i].s * spec[i].s : nullptr;
}


}  // namespace

extern "C" {

int tha4_ctx_create(int device, tha4_ctx** out) {
    if (!out) return THA4_ERR_INVALID;
    try {
        int count = 0;
        THA4_CUDA_CHECK(cudaGetDeviceCount(&count));
        THA4_REQUIRE(device >= 0 && device < count, "no such CUDA device");
        THA4_CUDA_CHECK(cudaSetDevice(device));
        cudaDeviceProp prop;
        THA4_CUDA_CHECK(cudaGetDeviceProperties(&prop, device));
        THA4_REQUIRE(prop.major == 9 && prop.minor == 0, "tha4_b200 is built for sm_90a (H100) only; found sm_" + std::to_string(prop.major) + std::to_string(prop.minor));
        auto* ctx = new tha4_ctx();
        ctx->device = device;
        THA4_CUDA_CHECK(cudaMalloc(&ctx->flag, sizeof(int)));
        THA4_CUDA_CHECK(cudaMalloc(&ctx->loss_acc, 4 * sizeof(double)));
        ctx->stats_cap = (size_t)32 << 20;                      // 32 Mi doubles = 256 MB (enough for micro-batches of 32)
        THA4_CUDA_CHECK(cudaMalloc(&ctx->stats_base, ctx->stats_cap * sizeof(double)));
        THA4_CUDA_CHECK(cudaMemset(ctx->stats_base, 0, ctx->stats_cap * sizeof(double)));
        ctx->decomposer.reset(new EncDecNet(TAIL_DECOMPOSER, 128, 4, 0));
        ctx->combiner.reset(new EncDecNet(TAIL_COMBINER, 128, 8, 12));
        ctx->face.reset(new EncDecNet(TAIL_FACE, 192, 4, 27));
        ctx->body.reset(new UNetNet(false, 256, 64, {1, 2, 4, 4, 4}));           // mode_07.py:210-226
        ctx->upscaler.reset(new UNetNet(true, 512, 32, {1, 2, 4, 8, 8, 8}));     // mode_07.py:241-257
        ctx->sface.reset(new SirenFaceNet());
        ctx->sbody.reset(new SirenBodyNet());
        *out = ctx;
        return THA4_OK;
    } catch (const CudaError& e) {
        g_create_err = e.what();
        return THA4_ERR_CUDA;
    } catch (const std::exception& e) {
        g_create_err = e.what();
        return THA4_ERR_INVALID;
    }
}

int tha4_ctx_destroy(tha4_ctx* ctx) {
    if (!ctx) return THA4_ERR_INVALID;
    cudaSetDevice(ctx->device);
    cudaDeviceSynchronize();
    if (ctx->flag) cudaFree(ctx->flag);
    if (ctx->loss_acc) cudaFree(ctx->loss_acc);
    if (ctx->pose_stage) cudaFree(ctx->pose_stage);
    if (ctx->capture_stream) cudaStreamDestroy(ctx->capture_stream);
    if (ctx->side) { cudaStreamDestroy(ctx->side); cudaEventDestroy(ctx->ev_fork); cudaEventDestroy(ctx->ev_join); }
    if (ctx->stats_base) cudaFree(ctx->stats_base);
    ctx->drop_graphs();
    delete ctx;
    return THA4_OK;
}

const char* tha4_last_error(const tha4_ctx* ctx) { return ctx ? ctx->err.c_str() : g_create_err.c_str(); }

int tha4_set_option(tha4_ctx* ctx, const char* name, int64_t value) {
    return guarded(ctx, [&] {
        cudaDeviceSynchronize();
        ctx->drop_graphs();                   // every option can change the launch sequence
        if (!strcmp(name, "strict")) { ctx->strict = value ? 1 : 0; }
        else if (!strcmp(name, "cuda_graphs")) ctx->use_graphs = value ? 1 : 0;
        else if (!strcmp(name, "side_stream")) ctx->side_streams = value ? 1 : 0;
        else if (!strcmp(name, "tcgen05")) conv_enable_tc(value != 0);
        else if (!strcmp(name, "cluster_splitk")) conv_tc_enable_cluster(value != 0);
        else if (!strcmp(name, "halo_conv")) conv_halo_enable(value != 0);
        else if (!strcmp(name, "tma_store")) conv_halo_enable_tma_store(value != 0);
        else if (!strcmp(name, "halo_m256")) { THA4_REQUIRE(value >= -1 && value <= 1, "halo_m256: -1, 0 or 1"); conv_halo_set_m256((int)value); }
        else if (!strcmp(name, "siren_tc")) siren_tc_enable(value != 0);
        else if (!strcmp(name, "tc_stride2")) conv_tc_enable_stride2(value != 0);
        else if (!strcmp(name, "small_bn")) conv_tc_enable_small_bn(value != 0);
        else if (!strcmp(name, "attn_split16")) attention_enable_split16(value != 0);
        else if (!strcmp(name, "tail_persist")) tail_tc_enable_persist(value != 0);
        else if (!strcmp(name, "attn_mma")) attention_enable_mma(value != 0);
        else if (!strcmp(name, "half_operands")) ctx->half_operands = value ? 1 : 0;
        else if (!strcmp(name, "pdl")) g_use_pdl = value != 0;
        else if (!strcmp(name, "profile")) { prof_enable(value != 0); if (value == 2) prof_reset(); }
        else if (!strcmp(name, "microbatch")) { THA4_REQUIRE(value >= 1 && value <= 1024, "microbatch range"); ctx->microbatch = (int)value; }
        else throw std::runtime_error(std::string("tha4: unknown option ") + name);
    });
}

int64_t tha4_get_counter(const tha4_ctx* ctx, const char* name) {
    if (!strcmp(name, "kernel_launches")) return g_kernel_launches.load();
    {   // "prof_<what>_<cat>": what in us|launches|flops|bytes, cat in conv|norm|tail|attn|glue|siren
        static const char* cats[] = {"conv", "norm", "tail", "attn", "glue", "siren"};
        static const char* whats[] = {"us", "launches", "flops", "bytes"};
        if (!strncmp(name, "prof_", 5))
            for (int w = 0; w < 4; ++w)
                for (int c = 0; c < 6; ++c)
                    if (std::string(name) == std::string("prof_") + whats[w] + "_" + cats[c]) {
                        try { return (int64_t)prof_read(c, w); } catch (...) { return -1; }
                    }
    }
    if (ctx && !strcmp(name, "graph_replays")) return (int64_t)ctx->graph_replays;
    if (ctx && !strcmp(name, "graph_captures")) return (int64_t)ctx->graph_captures;
    if (ctx && !strcmp(name, "graph_failures")) return (int64_t)ctx->graph_failures;
    if (ctx && !strcmp(name, "workspace_bytes")) return (int64_t)(ctx->persist.bytes() + ctx->scratch.bytes());
    return -1;
}

int tha4_load_net(tha4_ctx* ctx, int net, int n_tensors, const char* const* keys, const void* const* dev_ptrs,
                  const int64_t* shapes, const int* ndims, void* stream) {
    return guarded(ctx, [&] {
        StateDict sd = make_sd(n_tensors, keys, dev_ptrs, shapes, ndims);
        cudaStream_t s = (cudaStream_t)stream;
        cudaDeviceSynchronize();
        ctx->drop_graphs();                   // graphs hold pointers to the previous weights
        conv_set_pack_rounding(!ctx->strict);     // non-strict: weights are rounded to TF32 once, at pack time
        switch (net) {
            case THA4_NET_EYEBROW_DECOMPOSER: ctx->decomposer.reset(new EncDecNet(TAIL_DECOMPOSER, 128, 4, 0)); ctx->decomposer->load(sd, s); break;
            case THA4_NET_EYEBROW_MORPHING_COMBINER: ctx->combiner.reset(new EncDecNet(TAIL_COMBINER, 128, 8, 12)); ctx->combiner->load(sd, s); break;
            case THA4_NET_FACE_MORPHER: ctx->face.reset(new EncDecNet(TAIL_FACE, 192, 4, 27)); ctx->face->load(sd, s); break;
            case THA4_NET_BODY_MORPHER: ctx->body.reset(new UNetNet(false, 256, 64, {1, 2, 4, 4, 4})); ctx->body->load(sd, s); break;
            case THA4_NET_UPSCALER: ctx->upscaler.reset(new UNetNet(true, 512, 32, {1, 2, 4, 8, 8, 8})); ctx->upscaler->load(sd, s); break;
            case THA4_NET_SIREN_FACE_MORPHER: ctx->sface.reset(new SirenFaceNet()); ctx->sface->load(sd, s); break;
            case THA4_NET_SIREN_BODY_MORPHER: ctx->sbody.reset(new SirenBodyNet()); ctx->sbody->load(sd, s); break;
            default: throw std::runtime_error("tha4: unknown network id");
        }
    });
}

// ------------------------------------------------------------------------------------------------ module level
int tha4_eyebrow_decomposer_forward(tha4_ctx* ctx, const float* image, int B, float* const* outputs, void* stream) {
    return guarded(ctx, [&] {
        Runtime rt = make_rt(ctx, stream);
        for_chunks(ctx, B, ctx->microbatch, rt.stream, [&](int n0, int b) {
            float* o[6]; offset_outputs<6>(outputs, kEncDecDecomposer, n0, o);
            ctx->decomposer->forward(rt, make_img(image + (size_t)n0 * 4 * 128 * 128, b, 4, 128, 128), ImgView{}, nullptr, 0, o);
        });
    });
}

int tha4_eyebrow_morphing_combiner_forward(tha4_ctx* ctx, const float* background_layer, const float* eyebrow_layer,
                                           const float* pose, int pose_ld, int B, float* const* outputs, void* stream) {
    return guarded(ctx, [&] {
        Runtime rt = make_rt(ctx, stream);
        for_chunks(ctx, B, ctx->microbatch, rt.stream, [&](int n0, int b) {
            float* o[8]; offset_outputs<8>(outputs, kCombiner, n0, o);
            const size_t off = (size_t)n0 * 4 * 128 * 128;
            ctx->combiner->forward(rt, make_img(eyebrow_layer + off, b, 4, 128, 128), make_img(background_layer + off, b, 4, 128, 128),
                                   pose + (size_t)n0 * pose_ld, pose_ld, o);
        });
    });
}

int tha4_face_morpher_forward(tha4_ctx* ctx, const float* image, const float* pose, int pose_ld, int B,
                              float* const* outputs, void* stream) {
    return guarded(ctx, [&] {
        Runtime rt = make_rt(ctx, stream);
        for_chunks(ctx, B, ctx->microbatch, rt.stream, [&](int n0, int b) {
            float* o[8]; offset_outputs<8>(outputs, kFace, n0, o);
            ctx->face->forward(rt, make_img(image + (size_t)n0 * 4 * 192 * 192, b, 4, 192, 192), ImgView{},
                               pose + (size_t)n0 * pose_ld, pose_ld, o);
        });
    });
}

int tha4_eyebrow_decomposer_backward(tha4_ctx* ctx, const float* image, int B, const float* const* grad_outputs,
                                     float* d_image, void* stream) {
    return guarded(ctx, [&] {
        THA4_REQUIRE(d_image != nullptr, "decomposer backward: no gradient requested");
        Runtime rt = make_rt(ctx, stream);
        for_chunks(ctx, B, ctx->microbatch, rt.stream, [&](int n0, int b) {
            const float* g[6]; offset_grads<6>(grad_outputs, kEncDecDecomposer, n0, g);
            EncDecGrads eg; eg.grad_outputs = g; eg.d_image0 = d_image + (size_t)n0 * 4 * 128 * 128;
            ctx->decomposer->backward(rt, make_img(image + (size_t)n0 * 4 * 128 * 128, b, 4, 128, 128), ImgView{}, nullptr, 0, eg);
        });
    });
}

int tha4_eyebrow_morphing_combiner_backward(tha4_ctx* ctx, const float* background_layer, const float* eyebrow_layer,
                                            const float* pose, int pose_ld, int B, const float* const* grad_outputs,
                                            float* d_background_layer, float* d_eyebrow_layer, float* d_pose, void* stream) {
    return guarded(ctx, [&] {
        THA4_REQUIRE(d_background_layer || d_eyebrow_layer || d_pose, "combiner backward: no gradient requested");
        THA4_REQUIRE(pose_ld >= 12, "combiner backward: pose rows need at least 12 entries");
        Runtime rt = make_rt(ctx, stream);
        for_chunks(ctx, B, ctx->microbatch, rt.stream, [&](int n0, int b) {
            const float* g[8]; offset_grads<8>(grad_outputs, kCombiner, n0, g);
            const size_t off = (size_t)n0 * 4 * 128 * 128;
            EncDecGrads eg; eg.grad_outputs = g;
            eg.d_image0 = d_eyebrow_layer ? d_eyebrow_layer + off : nullptr;
            eg.d_image1 = d_background_layer ? d_background_layer + off : nullptr;
            eg.d_pose = d_pose ? d_pose + (size_t)n0 * 12 : nullptr; eg.d_pose_ld = 12;
            ctx->combiner->backward(rt, make_img(eyebrow_layer + off, b, 4, 128, 128), make_img(background_layer + off, b, 4, 128, 128),
                                    pose + (size_t)n0 * pose_ld, pose_ld, eg);
        });
    });
}

int tha4_face_morpher_backward(tha4_ctx* ctx, const float* image, const float* pose, int pose_ld, int B,
                               const float* const* grad_outputs, float* d_image, float* d_pose, void* stream) {
    return guarded(ctx, [&] {
        THA4_REQUIRE(d_image || d_pose, "face morpher backward: no gradient requested");
        THA4_REQUIRE(pose_ld >= 27, "face morpher backward: pose rows need at least 27 entries");
        Runtime rt = make_rt(ctx, stream);
        for_chunks(ctx, B, ctx->microbatch, rt.stream, [&](int n0, int b) {
            const float* g[8]; offset_grads<8>(grad_outputs, kFace, n0, g);
            EncDecGrads eg; eg.grad_outputs = g;
            eg.d_image0 = d_image ? d_image + (size_t)n0 * 4 * 192 * 192 : nullptr;
            eg.d_pose = d_pose ? d_pose + (size_t)n0 * 27 : nullptr; eg.d_pose_ld = 27;
            ctx->face->backward(rt, make_img(image + (size_t)n0 * 4 * 192 * 192, b, 4, 192, 192), ImgView{}, pose + (size_t)n0 * pose_ld,
                                pose_ld, eg);
        });
    });
}

int tha4_morpher_forward(tha4_ctx* ctx, const float* image, const float* pose, int pose_ld, int B,
                         float* const* outputs, void* stream) {
    return guarded(ctx, [&] {
        Runtime rt = make_rt(ctx, stream);
        OutSpec spec[5]; fill_unet_spec(spec, 256);
        for_chunks(ctx, B, ctx->microbatch, rt.stream, [&](int n0, int b) {
            float* o[5]; offset_outputs<5>(outputs, spec, n0, o);
            ctx->body->forward(rt, make_img(image + (size_t)n0 * 4 * 256 * 256, b, 4, 256, 256), nullptr, nullptr, 0,
                               pose + (size_t)n0 * pose_ld, pose_ld, o);
        });
    });
}

int tha4_morpher_backward(tha4_ctx* ctx, const float* image, const float* pose, int pose_ld, int B,
                          const float* const* grad_outputs, float* d_image, float* d_pose, void* stream) {
    return guarded(ctx, [&] {
        THA4_REQUIRE(d_image || d_pose, "morpher backward: no gradient requested");
        THA4_REQUIRE(pose_ld >= 6, "morpher backward: pose rows need at least 6 entries");
        Runtime rt = make_rt(ctx, stream);
        OutSpec spec[5]; fill_unet_spec(spec, 256);
        for_chunks(ctx, B, ctx->microbatch, rt.stream, [&](int n0, int b) {
            const float* g[5]; offset_grads<5>(grad_outputs, spec, n0, g);
            UNetGrads ug; ug.grad_outputs = g;
            ug.d_image = d_image ? d_image + (size_t)n0 * 4 * 256 * 256 : nullptr;
            ug.d_pose = d_pose ? d_pose + (size_t)n0 * 6 : nullptr; ug.d_pose_ld = 6;
            ctx->body->backward(rt, make_img(image + (size_t)n0 * 4 * 256 * 256, b, 4, 256, 256), nullptr, nullptr, 0,
                                pose + (size_t)n0 * pose_ld, pose_ld, ug);
        });
    });
}

int tha4_upscaler_backward(tha4_ctx* ctx, const float* rest_image, const float* coarse_posed_image, const float* coarse_grid_change,
                           int coarse_size, const float* pose, int pose_ld, int B, const float* const* grad_outputs,
                           float* d_rest_image, float* d_coarse_posed_image, float* d_coarse_grid_change, float* d_pose, void* stream) {
    return guarded(ctx, [&] {
        THA4_REQUIRE(d_rest_image || d_coarse_posed_image || d_coarse_grid_change || d_pose, "upscaler backward: no gradient requested");
        THA4_REQUIRE(coarse_size == 256 || coarse_size == 512, "upscaler backward: coarse_size must be 256 or 512");
        THA4_REQUIRE(pose_ld >= 6, "upscaler backward: pose rows need at least 6 entries");
        Runtime rt = make_rt(ctx, stream);
        OutSpec spec[5]; fill_unet_spec(spec, 512);
        const size_t hw = 512 * 512, chw = (size_t)coarse_size * coarse_size;
        for_chunks(ctx, B, std::min(ctx->microbatch, UPSCALER_BWD_MAX_BATCH), rt.stream, [&](int n0, int b) {
            const float* g[5]; offset_grads<5>(grad_outputs, spec, n0, g);
            UNetGrads ug; ug.grad_outputs = g;
            ug.d_image = d_rest_image ? d_rest_image + (size_t)n0 * 4 * hw : nullptr;
            ug.d_coarse_posed = d_coarse_posed_image ? d_coarse_posed_image + (size_t)n0 * 4 * chw : nullptr;
            ug.d_coarse_grid = d_coarse_grid_change ? d_coarse_grid_change + (size_t)n0 * 2 * chw : nullptr;
            ug.d_pose = d_pose ? d_pose + (size_t)n0 * 6 : nullptr; ug.d_pose_ld = 6;
            ctx->upscaler->backward(rt, make_img(rest_image + (size_t)n0 * 4 * hw, b, 4, 512, 512), coarse_posed_image + (size_t)n0 * 4 * chw,
                                    coarse_grid_change + (size_t)n0 * 2 * chw, coarse_size, pose + (size_t)n0 * pose_ld, pose_ld, ug);
        });
    });
}

int tha4_upscaler_forward(tha4_ctx* ctx, const float* rest_image, const float* coarse_posed_image,
                          const float* coarse_grid_change, int coarse_size, const float* pose, int pose_ld, int B,
                          float* const* outputs, void* stream) {
    return guarded(ctx, [&] {
        Runtime rt = make_rt(ctx, stream);
        OutSpec spec[5]; fill_unet_spec(spec, 512);
        for_chunks(ctx, B, ctx->microbatch, rt.stream, [&](int n0, int b) {
            float* o[5]; offset_outputs<5>(outputs, spec, n0, o);
            ctx->upscaler->forward(rt, make_img(rest_image + (size_t)n0 * 4 * 512 * 512, b, 4, 512, 512),
                                   coarse_posed_image + (size_t)n0 * 4 * coarse_size * coarse_size,
                                   coarse_grid_change + (size_t)n0 * 2 * coarse_size * coarse_size, coarse_size, pose + (size_t)n0 * pose_ld, pose_ld, o);
        });
    });
}

int tha4_siren_face_morpher_forward(tha4_ctx* ctx, const float* pose, int pose_ld, int B, float* output, void* stream) {
    return guarded(ctx, [&] {
        Runtime rt = make_rt(ctx, stream);
        begin_pass(ctx, (cudaStream_t)stream);
        ctx->sface->forward(rt, pose, pose_ld, B, output);
    });
}

int tha4_siren_morpher_forward(tha4_ctx* ctx, const float* image, const float* pose, int pose_ld, int B,
                               float* const* outputs, void* stream) {
    return guarded(ctx, [&] {
        Runtime rt = make_rt(ctx, stream);
        begin_pass(ctx, (cudaStream_t)stream);
        ctx->sbody->forward(rt, make_img(image, B, 4, 512, 512), pose, pose_ld, outputs);
    });
}

// ------------------------------------------------------------------------------------------------ poser level
int tha4_teacher_forward(tha4_ctx* ctx, int mode, const float* image, int64_t image_batch_stride, const float* pose, int B,
                         float* const* outputs, int eyebrow_morphed_image_index, const float* const* cached_decomposer, void* stream) {
    return guarded(ctx, [&] {
        THA4_REQUIRE(mode == 7 || mode == 12, "teacher mode must be 7 or 12");
        THA4_REQUIRE(image_batch_stride == 0 || image_batch_stride == 4L * 512 * 512, "image batch stride must be 0 (one image, B poses) or 4*512*512");
        const long img_sn = (long)image_batch_stride;
        Runtime rt = make_rt(ctx, stream);
        OutSpec spec[33];
        int n = 0;
        if (mode == 7) {
            fill_unet_spec(spec, 512); n = 5;
            spec[n++] = {4, 512};
            fill_unet_spec(spec + n, 256); n += 5;
        }
        for (int i = 0; i < 8; ++i) spec[n++] = kFace[i];
        for (int i = 0; i < 8; ++i) spec[n++] = kCombiner[i];
        for (int i = 0; i < 6; ++i) spec[n++] = kEncDecDecomposer[i];
        const int nout = n;
        auto run = [&](const float* img_p, const float* pose_p, float* const* outs, const float* const* cached_p) {
            for_chunks(ctx, B, ctx->microbatch, rt.stream, [&](int n0, int b) {
                float* o[33];
                for (int i = 0; i < nout; ++i) o[i] = outs[i] ? outs[i] + (size_t)n0 * spec[i].c * spec[i].s * spec[i].s : nullptr;
                const float* cd[6];
                if (cached_p)
                    for (int i = 0; i < 6; ++i) cd[i] = cached_p[i] + (size_t)n0 * kEncDecDecomposer[i].c * 128 * 128;
                teacher_chunk(ctx, rt, mode, img_p + (size_t)n0 * img_sn, img_sn, pose_p + (size_t)n0 * 45, b, o,
                              eyebrow_morphed_image_index, cached_p ? cd : nullptr);
            });
        };
        // ---- CUDA-graph path: single-chunk calls whose buffer addresses repeat ----
        cudaStream_t s = rt.stream;
        if (ctx->graph_pause > 0) --ctx->graph_pause;
        if (ctx->use_graphs && B <= ctx->microbatch && B <= 1024 && !prof_enabled() && ctx->graph_pause == 0) {
            if (!ctx->pose_stage) THA4_CUDA_CHECK(cudaMalloc(&ctx->pose_stage, 1024 * 45 * sizeof(float)));
            std::vector<uintptr_t> key;
            key.reserve(nout + 12);
            key.push_back((uintptr_t)mode); key.push_back((uintptr_t)B); key.push_back((uintptr_t)eyebrow_morphed_image_index);
            key.push_back((uintptr_t)img_sn); key.push_back((uintptr_t)image); key.push_back((uintptr_t)s);
            for (int i = 0; i < nout; ++i) key.push_back((uintptr_t)outputs[i]);
            for (int i = 0; i < 6; ++i) key.push_back(cached_decomposer ? (uintptr_t)cached_decomposer[i] : 0);
            ++ctx->graph_clock;
            auto it = ctx->graphs.find(key);
            if (it != ctx->graphs.end()) {
                TeacherGraph& g = it->second;
                // the arena must be clean when the graph starts; its own first memset only knows the dirt that preceded the capture
                if (ctx->stats_off > 0) THA4_CUDA_CHECK(cudaMemsetAsync(ctx->stats_base, 0, ctx->stats_off * sizeof(double), s));
                ctx->stats_off = 0;
                THA4_CUDA_CHECK(cudaMemcpyAsync(ctx->pose_stage, pose, (size_t)B * 45 * sizeof(float), cudaMemcpyDeviceToDevice, s));
                THA4_CUDA_CHECK(cudaGraphLaunch(g.exec, s));
                g_kernel_launches.fetch_add(g.launches);
                ctx->stats_off = g.stats_end;
                g.last_use = ctx->graph_clock;
                ctx->graph_misses = 0;
                ++ctx->graph_replays;
                return;
            }
            if (++ctx->graph_misses >= 64) { ctx->graph_misses = 0; ctx->graph_pause = 512; }   // buffers keep moving: eager for a while
            if (++ctx->graph_seen[key] >= 2) {           // second sight of this set of buffers: worth a capture
                ctx->graph_seen.erase(key);
                const long l0 = g_kernel_launches.load();
                cudaGraph_t graph = nullptr;
                cudaGraphExec_t exec = nullptr;
                THA4_CUDA_CHECK(cudaMemcpyAsync(ctx->pose_stage, pose, (size_t)B * 45 * sizeof(float), cudaMemcpyDeviceToDevice, s));
                std::string why;
                cudaStream_t cap = s;
                if (s == nullptr || s == cudaStreamLegacy || s == cudaStreamPerThread) {
                    if (!ctx->capture_stream) THA4_CUDA_CHECK(cudaStreamCreateWithFlags(&ctx->capture_stream, cudaStreamNonBlocking));
                    cap = ctx->capture_stream;
                }
                cudaError_t e = cudaStreamBeginCapture(cap, cudaStreamCaptureModeThreadLocal);
                bool ok = e == cudaSuccess;
                if (!ok) why = std::string("begin: ") + cudaGetErrorString(e);
                if (ok) {
                    rt.stream = cap;
                    try { run(image, ctx->pose_stage, outputs, cached_decomposer); }
                    catch (const std::exception& ex) { ok = false; why = std::string("launch: ") + ex.what(); }
                    rt.stream = s;
                    e = cudaStreamEndCapture(cap, &graph);
                    if (e != cudaSuccess || graph == nullptr) { if (ok) why = std::string("end: ") + cudaGetErrorString(e); ok = false; }
                }
                if (ok) { e = cudaGraphInstantiate(&exec, graph, 0); if (e != cudaSuccess) { ok = false; why = std::string("instantiate: ") + cudaGetErrorString(e); } }
                if (graph) cudaGraphDestroy(graph);
                if (!ok) {                               // not capturable here: run this call eagerly, stop trying for a while
                    if (ctx->graph_failures++ == 0) fprintf(stderr, "tha4: CUDA graph capture failed (%s); launching eagerly\n", why.c_str());
                    cudaGetLastError();
                    ctx->graph_misses = 0; ctx->graph_pause = 512;
                    ctx->persist.reset(); ctx->scratch.reset();
                } else {
                    if ((int)ctx->graphs.size() >= GRAPH_CACHE) {
                        auto victim = ctx->graphs.begin();
                        for (auto jt = ctx->graphs.begin(); jt != ctx->graphs.end(); ++jt)
                            if (jt->second.last_use < victim->second.last_use) victim = jt;
                        cudaGraphExecDestroy(victim->second.exec);
                        ctx->graphs.erase(victim);
                    }
                    TeacherGraph g;
                    g.exec = exec; g.launches = g_kernel_launches.load() - l0; g.stats_end = ctx->stats_off; g.last_use = ctx->graph_clock;
                    ctx->graphs[key] = g;
                    ++ctx->graph_captures;
                    // the capture recorded the work without running it: replay it now for this call
                    THA4_CUDA_CHECK(cudaGraphLaunch(exec, s));
                    return;
                }
            }
            if (ctx->graph_seen.size() > 256) ctx->graph_seen.clear();
        }
        run(image, pose, outputs, cached_decomposer);
    });
}

int tha4_student_forward(tha4_ctx* ctx, const float* image, const float* pose, int B, float* const* outputs, void* stream) {
    return guarded(ctx, [&] {
        Runtime rt = make_rt(ctx, stream);
        cudaStream_t s = rt.stream;
        begin_pass(ctx, (cudaStream_t)stream);
        // face SIREN from pose[:, :39] (mode_14.py:64-71), pasted at rows 80:208, cols 192:320 (:72-78)
        ctx->sface->forward(rt, pose, 45, B, outputs[5]);
        float* body_in = ctx->persist.alloc((size_t)B * 4 * 512 * 512);
        copy_window(make_img(image, B, 4, 512, 512), body_in, 4L * 512 * 512, 512L * 512, 512, s);
        copy_window(make_img(outputs[5], B, 4, 128, 128), body_in + 80 * 512 + 192, 4L * 512 * 512, 512L * 512, 512, s);
        ctx->sbody->forward(rt, make_img(body_in, B, 4, 512, 512), pose, 45, outputs);
    });
}

int tha4_student_forward_io(tha4_ctx* ctx, const void* image, const float* pose, int B, void* const* outputs, int io_dtype, void* stream) {
    if (io_dtype == 0) return tha4_student_forward(ctx, (const float*)image, pose, B, (float* const*)outputs, stream);
    return guarded(ctx, [&] {
        THA4_REQUIRE(io_dtype == 1, "student forward: io_dtype must be 0 (fp32) or 1 (fp16)");
        Runtime rt = make_rt(ctx, stream);
        cudaStream_t s = rt.stream;
        begin_pass(ctx, (cudaStream_t)stream);
        // fp16 image in, fp16 planes out; the sampled image and the face patch stay fp32 inside (the gather reads them four
        // times per pixel from L2, the conversion is one pass over 4 MB per frame)
        const long img_n = (long)B * 4 * 512 * 512, face_n = (long)B * 4 * 128 * 128;
        float* body_in = ctx->persist.alloc((size_t)img_n);
        float* face32 = ctx->persist.alloc((size_t)face_n);
        ctx->sface->forward(rt, pose, 45, B, face32);
        convert_flat_f32((const __half*)image, body_in, img_n, s);
        copy_window(make_img(face32, B, 4, 128, 128), body_in + 80 * 512 + 192, 4L * 512 * 512, 512L * 512, 512, s);
        convert_flat_f16(face32, (__half*)outputs[5], face_n, s);
        ctx->sbody->forward(rt, make_img(body_in, B, 4, 512, 512), pose, 45, (float* const*)outputs, true);
    });
}

int64_t tha4_siren_morpher_param_count(void) { return (int64_t)siren_body_param_count(); }

int tha4_siren_morpher_train_step(tha4_ctx* ctx, const float* image, const float* pose, const float* target_posed,
                                  const float* target_warped, const float* target_grid_change, const float* loss_weights,
                                  const float* params, float* grads, double* host_loss_means, int B, void* stream) {
    return guarded(ctx, [&] {
        THA4_REQUIRE(B >= 1 && B <= 8, "distill step: per-GPU batch must be 1..8 (distiller_config.py:100-104)");
        cudaStream_t s = (cudaStream_t)stream;
        begin_pass(ctx, s);
        Runtime rt = make_rt(ctx, stream);
        siren_body_train_step(rt, make_img(image, B, 4, 512, 512), pose, 45, target_posed, target_warped, target_grid_change,
                              loss_weights, params, grads, ctx->loss_acc);
        if (host_loss_means) {
            double h[4];
            THA4_CUDA_CHECK(cudaMemcpyAsync(h, ctx->loss_acc, sizeof(h), cudaMemcpyDeviceToHost, s));
            THA4_CUDA_CHECK(cudaStreamSynchronize(s));
            const double nb = (double)B * 4 * 512 * 512, ng = (double)B * 2 * 512 * 512;
            host_loss_means[0] = h[0] / nb; host_loss_means[1] = h[1] / nb; host_loss_means[2] = h[2] / ng; host_loss_means[3] = h[3] / nb;
        }
    });
}

int64_t tha4_siren_face_morpher_param_count(void) { return (int64_t)siren_face_param_count(); }

int tha4_siren_face_morpher_train_step(tha4_ctx* ctx, const float* pose, int pose_ld, const float* target, const float* mask,
                                       const float* loss_weights, const float* params, float* grads, double* host_loss_means,
                                       int B, void* stream) {
    return guarded(ctx, [&] {
        THA4_REQUIRE(B >= 1 && B <= 64, "face distill step: per-GPU batch must be 1..64");
        THA4_REQUIRE(pose_ld >= 39, "face distill step: pose rows need at least 39 entries");
        cudaStream_t s = (cudaStream_t)stream;
        begin_pass(ctx, s);
        Runtime rt = make_rt(ctx, stream);
        siren_face_train_step(rt, pose, pose_ld, B, target, mask, loss_weights, params, grads, ctx->loss_acc);
        if (host_loss_means) {
            double h[2];
            THA4_CUDA_CHECK(cudaMemcpyAsync(h, ctx->loss_acc, sizeof(h), cudaMemcpyDeviceToHost, s));
            THA4_CUDA_CHECK(cudaStreamSynchronize(s));
            const double nel = (double)B * 4 * 128 * 128;
            host_loss_means[0] = h[0] / nel; host_loss_means[1] = h[1] / nel;
        }
    });
}

int tha4_siren_morpher_backward(tha4_ctx* ctx, const float* image, const float* pose, int pose_ld, int B,
                                const float* const* grad_outputs, const float* grid_change, const float* alpha,
                                const float* params, float* grads, float* d_image, float* d_pose, void* stream) {
    return guarded(ctx, [&] {
        THA4_REQUIRE(B >= 1, "student backward: batch must be >= 1");
        THA4_REQUIRE(grads || d_image || d_pose, "student backward: no output requested");
        const bool siren = grads || d_pose;          // the parameter and pose gradients need the SIREN recompute; d_image does not
        THA4_REQUIRE(!siren || (image && pose && params), "student backward: image, pose and params are required");
        THA4_REQUIRE(!siren || pose_ld >= 45, "student backward: pose rows need at least 45 entries");
        THA4_REQUIRE(!d_image || (grid_change && alpha), "student backward: d_image needs the forward's grid_change and alpha");
        Runtime rt = make_rt(ctx, stream);
        if (grads) THA4_CUDA_CHECK(cudaMemsetAsync(grads, 0, siren_body_param_count() * sizeof(float), rt.stream));
        constexpr size_t hw = 512 * 512;
        for_chunks(ctx, B, SIREN_BODY_MAX_BATCH, rt.stream, [&](int n0, int b) {     // micro-batches accumulate into grads
            const float* g[5]; offset_grads<5>(grad_outputs, kSirenBody, n0, g);
            if (siren)
                siren_body_backward(rt, make_img(image + (size_t)n0 * 4 * hw, b, 4, 512, 512), pose + (size_t)n0 * pose_ld, pose_ld, g,
                                    params, grads, d_pose ? d_pose + (size_t)n0 * 45 : nullptr);
            if (d_image)
                siren_body_image_grad(rt, grid_change + (size_t)n0 * 2 * hw, alpha + (size_t)n0 * hw, g[0], g[3], b,
                                      d_image + (size_t)n0 * 4 * hw);
        });
    });
}

int tha4_siren_face_morpher_backward(tha4_ctx* ctx, const float* pose, int pose_ld, int B, const float* grad_output,
                                     const float* params, float* grads, float* d_pose, void* stream) {
    return guarded(ctx, [&] {
        THA4_REQUIRE(B >= 1, "face student backward: batch must be >= 1");
        THA4_REQUIRE(grads || d_pose, "face student backward: no output requested");
        THA4_REQUIRE(pose_ld >= 39, "face student backward: pose rows need at least 39 entries");
        THA4_REQUIRE(grad_output != nullptr, "face student backward: grad_output is required");
        Runtime rt = make_rt(ctx, stream);
        if (grads) THA4_CUDA_CHECK(cudaMemsetAsync(grads, 0, siren_face_param_count() * sizeof(float), rt.stream));
        for_chunks(ctx, B, SIREN_FACE_MAX_BATCH, rt.stream, [&](int n0, int b) {     // micro-batches accumulate into grads
            siren_face_backward(rt, pose + (size_t)n0 * pose_ld, pose_ld, b, grad_output + (size_t)n0 * 4 * 128 * 128, params, grads,
                                d_pose ? d_pose + (size_t)n0 * 39 : nullptr);
        });
    });
}

int tha4_adam_step(tha4_ctx* ctx, float* params, const float* grads, float* exp_avg, float* exp_avg_sq, int64_t n, float lr,
                   float beta1, float beta2, float eps, int step, float grad_scale, void* stream) {
    return guarded(ctx, [&] { adam_step(params, grads, exp_avg, exp_avg_sq, (long)n, lr, beta1, beta2, eps, step, grad_scale, (cudaStream_t)stream); });
}

int tha4_images_differ(tha4_ctx* ctx, const float* a, const float* b, int64_t n, int* differ, void* stream) {
    return guarded(ctx, [&] { *differ = images_differ(a, b, (size_t)n, ctx->flag, (cudaStream_t)stream) ? 1 : 0; });
}

int tha4_frame_to_srgb8(tha4_ctx* ctx, const float* frame, int B, int H, int W, int background, int round_mode, uint8_t* out, void* stream) {
    return guarded(ctx, [&] { frame_to_srgb8(frame, B, H, W, background, round_mode, out, (cudaStream_t)stream); });
}

int tha4_rgba8_to_poser_image(tha4_ctx* ctx, const uint8_t* rgba, int H, int W, float* out, void* stream) {
    return guarded(ctx, [&] { rgba8_to_poser_image(rgba, H, W, out, (cudaStream_t)stream); });
}

// ------------------------------------------------------------------------------------------------ kernel level
int tha4_grid_sample(tha4_ctx* ctx, const float* image, const float* grid_change, int N, int C, int H, int W,
                     float* out, int32_t* x0, int32_t* y0, float* tx, float* ty, void* stream) {
    return guarded(ctx, [&] { grid_sample(make_img(image, N, C, H, W), grid_change, out, x0, y0, tx, ty, (cudaStream_t)stream); });
}

int tha4_resize_bilinear(tha4_ctx* ctx, const float* in, int N, int C, int Hi, int Wi, int Ho, int Wo, float* out, void* stream) {
    return guarded(ctx, [&] { resize_bilinear(make_img(in, N, C, Hi, Wi), out, Ho, Wo, (cudaStream_t)stream); });
}

int tha4_base_grid(int size, float* host_out) {
    if (size < 2 || !host_out) return THA4_ERR_INVALID;
    base_grid_host(size, host_out);
    return THA4_OK;
}

int tha4_test_conv(tha4_ctx* ctx, int kind, const float* x, const float* w, const float* bias, const float* res,
                   int res_mode, int in_up, float* y, int N, int Cin, int H, int W, int Cout, int strict, int ksplit,
                   void* stream) {
    return guarded(ctx, [&] {
        cudaStream_t s = (cudaStream_t)stream;
        begin_pass(ctx, (cudaStream_t)stream);
        Pool* P = &ctx->persist;
        const int cin_k = round_up(Cin, 4);
        ConvWeights cw;
        conv_describe(cw, (ConvKind)kind, cin_k, Cout);
        conv_set_pack_rounding(!strict);
        cw.tf32_rounded = !strict;
        cw.w = P->alloc(conv_packed_floats(cw));
        THA4_CUDA_CHECK(cudaMemsetAsync(cw.w, 0, conv_packed_floats(cw) * sizeof(float), s));
        conv_pack(cw, (ConvKind)kind, w, Cin, 0, s);
        cw.bias = const_cast<float*>(bias);
        auto mk = [&](int h, int ww, int c) { View v; v.N = N; v.H = h; v.W = ww; v.C = c; v.ld = c; v.p = P->alloc((size_t)N * h * ww * c); return v; };
        View xin = mk(H, W, cin_k);
        if (cin_k != Cin) THA4_CUDA_CHECK(cudaMemsetAsync(xin.p, 0, xin.pixels() * cin_k * sizeof(float), s));
        nchw_to_nhwc(make_img(x, N, Cin, H, W), xin.slice(0, Cin), s);
        const int LH = in_up ? 2 * H : H, LW = in_up ? 2 * W : W;
        const bool x2 = (kind == CONVT_4x4_S2 || kind == CONV_UP2_3x3);
        const int Ho = (kind == CONV_4x4_S2) ? LH / 2 : (x2 ? LH * 2 : LH);
        const int Wo = (kind == CONV_4x4_S2) ? LW / 2 : (x2 ? LW * 2 : LW);
        View yo = mk(Ho, Wo, Cout);
        ConvArgs a;
        a.in = xin; a.in_up = in_up; a.out = yo; a.strict = strict; a.ksplit = ksplit;
        if (ctx->half_operands && !strict && conv_tc_enabled() && cin_k % 8 == 0 && conv_tc_supported(cw, a)) {
            // exercise the f16-operand variant the networks use between a normalisation layer and a conv
            View x16 = xin; x16.f16 = 1; x16.p = P->alloc((xin.pixels() * cin_k + 1) / 2);
            convert_f16(xin, x16, s);
            a.in = x16;
        }
        if (res) {
            const int rh = res_mode == RES_UP2 ? Ho / 2 : (res_mode == RES_DOWN2 ? Ho * 2 : Ho);
            const int rw = res_mode == RES_UP2 ? Wo / 2 : (res_mode == RES_DOWN2 ? Wo * 2 : Wo);
            View r = mk(rh, rw, Cout);
            nchw_to_nhwc(make_img(res, N, Cout, rh, rw), r, s);
            a.res = r; a.res_mode = res_mode;
        }
        const size_t wsf = conv_workspace_floats(cw, a);
        if (wsf) { a.ws = ctx->scratch.alloc(wsf); a.ws_floats = wsf; }
        conv_forward(cw, a, s);
        nhwc_to_nchw(yo, y, s);
        if (cw.w16) { THA4_CUDA_CHECK(cudaStreamSynchronize(s)); cudaFree(cw.w16); cw.w16 = nullptr; }   // made on first use, owned by this call
    });
}

static int test_conv_norm(tha4_ctx* ctx, int kind, const float* x, int N, int Cin, int H, int W, int norm_C, int groups,
                          const float* gamma, const float* beta, const float* film0, const float* film1, int act,
                          const float* w, const float* bias, const float* res, int res_mode, int Cout, int ksplit,
                          float* y, float* y_from_f16, double* y_stats, int reps, float* us_per_launch, void* stream) {
    return guarded(ctx, [&] {
        cudaStream_t s = (cudaStream_t)stream;
        begin_pass(ctx, s);
        Runtime rt = make_rt(ctx, stream);
        Pool* P = &ctx->persist;
        THA4_REQUIRE(Cin % 8 == 0 && norm_C % 8 == 0 && norm_C <= Cin, "test_conv_norm: channel counts must be multiples of 8");
        AllocSink sink;
        ConvWeights cw;
        {
            SinkScope own(&sink);
            conv_describe(cw, (ConvKind)kind, Cin, Cout);
            conv_set_pack_rounding(true);
            cw.tf32_rounded = true;
            cw.w = reinterpret_cast<float*>(tracked_malloc(conv_packed_floats(cw) * sizeof(float)));
            THA4_CUDA_CHECK(cudaMemsetAsync(cw.w, 0, conv_packed_floats(cw) * sizeof(float), s));
            conv_pack(cw, (ConvKind)kind, w, Cin, 0, s);
            conv_make_half(cw, s);
        }
        cw.bias = const_cast<float*>(bias);
        auto mk = [&](int n, int h, int ww, int c) { View v; v.N = n; v.H = h; v.W = ww; v.C = c; v.ld = c; v.p = P->alloc((size_t)n * h * ww * c); return v; };
        // raw input: fp32 (for the statistics, as a producing conv's fp32 accumulators would give them) + its f16 copy
        View xin = mk(N, H, W, Cin);
        xin.stats_rep = 2; xin.stats_rep_stride = (long)N * Cin * 2;
        xin.stats = rt.alloc_stats((size_t)2 * N * Cin * 2); xin.stats_ld = Cin;
        nchw_to_nhwc(make_img(x, N, Cin, H, W), xin, s);
        norm_stats(xin, s);
        View x16 = xin; x16.f16 = 1; x16.stats = nullptr; x16.p = P->alloc(((size_t)N * H * W * Cin + 1) / 2);
        convert_f16(xin, x16, s);
        const bool x2 = (kind == CONVT_4x4_S2 || kind == CONV_UP2_3x3);
        const int Ho = (kind == CONV_4x4_S2) ? H / 2 : (x2 ? H * 2 : H), Wo = (kind == CONV_4x4_S2) ? W / 2 : (x2 ? W * 2 : W);
        View yo = mk(N, Ho, Wo, Cout);
        if (y_stats) {        // per-(n, c) sum / sum of squares of the output, one replica
            yo.stats = rt.alloc_stats((size_t)N * Cout * 2); yo.stats_ld = Cout; yo.stats_rep = 1; yo.stats_rep_stride = (long)N * Cout * 2;
            THA4_CUDA_CHECK(cudaMemsetAsync(yo.stats, 0, (size_t)N * Cout * 2 * sizeof(double), s));
        }
        View y16 = yo; y16.f16 = 1; y16.stats = nullptr; y16.p = P->alloc(((size_t)N * Ho * Wo * Cout + 1) / 2);
        ConvArgs a;
        a.in = x16; a.out = yo; a.out16 = y16; a.ksplit = ksplit;
        a.nin.on = norm_C > 0; a.nin.C = norm_C; a.nin.groups = groups; a.nin.act = act == ACT_SILU ? ACT_SILU_FAST : act;
        a.nin.gamma = gamma; a.nin.beta = beta; a.nin.film0 = film0; a.nin.film1 = film1; a.nin.film1_ld = 2 * norm_C;
        a.nin.stats = xin.stats; a.nin.stats_ld = xin.stats_ld; a.nin.stats_rep = xin.stats_rep; a.nin.stats_rep_stride = xin.stats_rep_stride;
        if (res) {
            const int rh = res_mode == RES_UP2 ? Ho / 2 : (res_mode == RES_DOWN2 ? Ho * 2 : Ho);
            const int rw = res_mode == RES_UP2 ? Wo / 2 : (res_mode == RES_DOWN2 ? Wo * 2 : Wo);
            View r = mk(N, rh, rw, Cout);
            nchw_to_nhwc(make_img(res, N, Cout, rh, rw), r, s);
            a.res = r; a.res_mode = res_mode;
        }
        const size_t wsf = conv_workspace_floats(cw, a);
        if (wsf) { a.ws = ctx->scratch.alloc(wsf); a.ws_floats = wsf; }
        conv_forward(cw, a, s);
        if (y_stats) THA4_CUDA_CHECK(cudaMemcpyAsync(y_stats, yo.stats, (size_t)N * Cout * 2 * sizeof(double), cudaMemcpyDeviceToDevice, s));
        if (getenv("THA4_HALO_DEBUG")) { conv_forward(cw, a, s); conv_halo_debug_dump(); }
        if (reps > 0) {       // device time of the conv alone: `reps` back-to-back launches between two events
            cudaEvent_t e0, e1;
            THA4_CUDA_CHECK(cudaEventCreate(&e0)); THA4_CUDA_CHECK(cudaEventCreate(&e1));
            THA4_CUDA_CHECK(cudaEventRecord(e0, s));
            for (int i = 0; i < reps; ++i) conv_forward(cw, a, s);
            THA4_CUDA_CHECK(cudaEventRecord(e1, s));
            THA4_CUDA_CHECK(cudaEventSynchronize(e1));
            float ms = 0.0f;
            THA4_CUDA_CHECK(cudaEventElapsedTime(&ms, e0, e1));
            cudaEventDestroy(e0); cudaEventDestroy(e1);
            if (us_per_launch) *us_per_launch = 1000.0f * ms / reps;
        }
        nhwc_to_nchw(yo, y, s);
        if (y_from_f16) {
            View back = mk(N, Ho, Wo, Cout);
            convert_f32(y16, back, s);
            nhwc_to_nchw(back, y_from_f16, s);
        }
        THA4_CUDA_CHECK(cudaStreamSynchronize(s));
    });
}

int tha4_test_conv_norm(tha4_ctx* ctx, int kind, const float* x, int N, int Cin, int H, int W, int norm_C, int groups,
                        const float* gamma, const float* beta, const float* film0, const float* film1, int act,
                        const float* w, const float* bias, const float* res, int res_mode, int Cout, int ksplit,
                        float* y, float* y_from_f16, void* stream) {
    return test_conv_norm(ctx, kind, x, N, Cin, H, W, norm_C, groups, gamma, beta, film0, film1, act, w, bias, res, res_mode, Cout,
                          ksplit, y, y_from_f16, nullptr, 0, nullptr, stream);
}

int tha4_test_conv_norm_ex(tha4_ctx* ctx, int kind, const float* x, int N, int Cin, int H, int W, int norm_C, int groups,
                           const float* gamma, const float* beta, const float* film0, const float* film1, int act,
                           const float* w, const float* bias, const float* res, int res_mode, int Cout, int ksplit,
                           float* y, float* y_from_f16, double* y_stats, int reps, float* us_per_launch, void* stream) {
    return test_conv_norm(ctx, kind, x, N, Cin, H, W, norm_C, groups, gamma, beta, film0, film1, act, w, bias, res, res_mode, Cout,
                          ksplit, y, y_from_f16, y_stats, reps, us_per_launch, stream);
}

int tha4_test_norm(tha4_ctx* ctx, const float* x, int N, int C, int H, int W, int groups, const float* gamma,
                   const float* beta, const float* film0, const float* film1, int act, int pool, int out_f16, float* y, void* stream) {
    return guarded(ctx, [&] {
        cudaStream_t s = (cudaStream_t)stream;
        begin_pass(ctx, s);
        Runtime rt = make_rt(ctx, stream);
        Pool* P = &ctx->persist;
        View xin; xin.N = N; xin.H = H; xin.W = W; xin.C = C; xin.ld = C; xin.p = P->alloc((size_t)N * H * W * C);
        xin.stats_rep = 2; xin.stats_rep_stride = (long)N * C * 2;
        xin.stats = rt.alloc_stats((size_t)2 * N * C * 2); xin.stats_ld = C;
        nchw_to_nhwc(make_img(x, N, C, H, W), xin, s);
        norm_stats(xin, s);
        View yo = xin; yo.stats = nullptr;
        if (pool) { yo.H = H / 2; yo.W = W / 2; }
        yo.p = P->alloc((size_t)N * yo.H * yo.W * C);
        if (out_f16) {     // the variant the default mode runs: f16 output (operand of a wgmma conv), fast-math SiLU
            View y16 = yo; y16.f16 = 1; y16.p = P->alloc(((size_t)N * yo.H * yo.W * C + 1) / 2);
            norm_apply_fused(xin, groups, gamma, beta, film0, film1, 2 * C, act == ACT_SILU ? ACT_SILU_FAST : act, pool, nullptr, y16, s, 1);
            convert_f32(y16, yo, s);
        } else {
            norm_apply_fused(xin, groups, gamma, beta, film0, film1, 2 * C, act, pool, nullptr, yo, s, 0);
        }
        nhwc_to_nchw(yo, y, s);
    });
}

int tha4_test_tail(tha4_ctx* ctx, int kind, const float* feature, int N, int C, int S, const float* gamma, const float* beta,
                   int groups, int act, const float* head_w, const float* head_b, const int* head_cout, int n_heads,
                   const float* image0, const float* image1, float* const* outputs, int strict, void* stream) {
    return guarded(ctx, [&] {
        cudaStream_t s = (cudaStream_t)stream;
        begin_pass(ctx, s);
        Runtime rt = make_rt(ctx, stream);
        rt.strict = strict;
        Pool* P = &ctx->persist;
        View f; f.N = N; f.H = S; f.W = S; f.C = C; f.ld = C; f.p = P->alloc((size_t)N * S * S * C);
        f.stats_rep = 2; f.stats_rep_stride = (long)N * C * 2;
        f.stats = rt.alloc_stats((size_t)2 * N * C * 2); f.stats_ld = C;
        nchw_to_nhwc(make_img(feature, N, C, S, S), f, s);
        norm_stats(f, s);
        float* coef = P->alloc((size_t)N * C * 2);
        norm_finalize(f, groups, gamma, beta, nullptr, nullptr, 0, coef, s);
        AllocSink sink;
        TailWeights tw;
        {
            SinkScope own(&sink);
            tail_init(tw, C, s);
            size_t woff = 0, boff = 0;
            for (int i = 0; i < n_heads; ++i) {
                const bool has_b = head_b != nullptr && !((kind == TAIL_COMBINER || kind == TAIL_FACE) && i == 0);   // grid_change heads have no bias
                tail_add(tw, head_w + woff, has_b ? head_b + boff : nullptr, head_cout[i], s);
                woff += (size_t)head_cout[i] * C * 9; boff += head_cout[i];
            }
        }
        const int a = (act == ACT_SILU && !strict) ? ACT_SILU_FAST : act;
        const ImgView i0 = make_img(image0, N, 4, S, S);
        const ImgView i1 = image1 ? make_img(image1, N, 4, S, S) : ImgView{};
        if (!strict && rt.f16) {      // the default mode's kernel: raw f16 feature map + statistics -> wgmma tail
            { SinkScope own(&sink); tail_make_half(tw, s); }
            View f16v = f; f16v.f16 = 1; f16v.p = P->alloc(((size_t)N * S * S * C + 1) / 2);
            convert_f16(f, f16v, s);
            NormSpecTail ns; ns.groups = groups; ns.act = a; ns.gamma = gamma; ns.beta = beta;
            // interleaved copies of the image(s), as the networks hand them over (their own NHWC input tensors)
            View g0; g0.N = N; g0.H = S; g0.W = S; g0.C = 4; g0.ld = 4; g0.p = P->alloc((size_t)N * S * S * 4);
            nchw_to_nhwc(i0, g0, s);
            View g1 = g0;
            if (image1) { g1.p = P->alloc((size_t)N * S * S * 4); nchw_to_nhwc(i1, g1, s); }
            tail_tc_forward((TailKind)kind, tw, f16v, ns, i0, i1, outputs, s, &g0, image1 ? &g1 : nullptr);
        } else {
            tail_forward((TailKind)kind, tw, f, coef, a, i0, i1, outputs, s, strict);
        }
        THA4_CUDA_CHECK(cudaStreamSynchronize(s));       // `sink` frees the head weights on return
    });
}

int tha4_test_conv_backward_data(tha4_ctx* ctx, int kind, const float* dy, const float* w, float* dx, int N, int Cin, int H, int W,
                                 int Cout, int strict, void* stream) {
    return guarded(ctx, [&] {
        cudaStream_t s = (cudaStream_t)stream;
        begin_pass(ctx, s);
        THA4_REQUIRE(kind >= 0 && kind <= 5 && Cout % 4 == 0 && (kind == 0 || kind == 5 || Cin % 4 == 0),
                     "test_conv_backward_data: kind 0..5, Cout % 4 == 0 (and Cin % 4 == 0 for kinds 1..4)");
        const bool packed = kind >= 3;        // kind 5: a 3x3 conv through the packed forward weights (Cin zero-padded to 4)
        if (kind == 5) kind = CONV_3x3;
        Runtime rt = make_rt(ctx, stream);
        rt.strict = strict;
        Pool* P = &ctx->persist;
        AllocSink sink;
        ConvWeights cw;
        {
            SinkScope own(&sink);
            conv_set_pack_rounding(!strict);
            if (!packed) {
                conv_pack_adjoint(cw, (ConvKind)kind, w, Cin, Cout, kind == CONV_3x3 ? round_up(Cin, 4) : 0, s);
            } else {   // the U-Net's path: the forward conv packed as the network packs it, its adjoint made from the packed weights
                ConvWeights fwd;
                conv_describe(fwd, (ConvKind)kind, round_up(Cin, 4), Cout);
                fwd.w = reinterpret_cast<float*>(tracked_malloc(conv_packed_floats(fwd) * sizeof(float)));
                THA4_CUDA_CHECK(cudaMemsetAsync(fwd.w, 0, conv_packed_floats(fwd) * sizeof(float), s));
                conv_pack(fwd, (ConvKind)kind, w, Cin, 0, s);
                fwd.tf32_rounded = !strict;
                conv_adjoint_from_packed(cw, fwd, (ConvKind)kind, s);
            }
        }
        const int cin_k = kind == CONV_3x3 ? round_up(Cin, 4) : Cin;
        const int Ho = kind == 1 ? H / 2 : ((kind == 2 || kind == 4) ? 2 * H : H), Wo = kind == 1 ? W / 2 : ((kind == 2 || kind == 4) ? 2 * W : W);
        auto mk = [&](int h, int ww, int c) { View v; v.N = N; v.H = h; v.W = ww; v.C = c; v.ld = c; v.p = P->alloc((size_t)N * h * ww * c); return v; };
        View g = mk(Ho, Wo, Cout);
        nchw_to_nhwc(make_img(dy, N, Cout, Ho, Wo), g, s);
        View o = mk(H, W, cin_k);
        ConvArgs a;
        a.in = g; a.out = o; a.strict = strict;
        const size_t wsf = conv_workspace_floats(cw, a);
        if (wsf) { a.ws = ctx->scratch.alloc(wsf); a.ws_floats = wsf; }
        conv_forward(cw, a, s);
        nhwc_to_nchw(o.slice(0, Cin), dx, s);
        THA4_CUDA_CHECK(cudaStreamSynchronize(s));       // `sink` frees the packed weights on return
    });
}

int tha4_test_norm_backward(tha4_ctx* ctx, const float* x, int N, int C, int H, int W, const float* gamma, const float* beta,
                            int act, const float* dy, float* dx, void* stream) {
    return guarded(ctx, [&] {
        cudaStream_t s = (cudaStream_t)stream;
        begin_pass(ctx, s);
        Runtime rt = make_rt(ctx, stream);
        Pool* P = &ctx->persist;
        auto mk = [&](int c) { View v; v.N = N; v.H = H; v.W = W; v.C = c; v.ld = c; v.p = P->alloc((size_t)N * H * W * c); return v; };
        View xin = mk(C);
        xin.stats_rep = 2; xin.stats_rep_stride = (long)N * C * 2;
        xin.stats = rt.alloc_stats((size_t)2 * N * C * 2); xin.stats_ld = C;
        nchw_to_nhwc(make_img(x, N, C, H, W), xin, s);
        norm_stats(xin, s);
        View g = mk(C), o = mk(C);
        nchw_to_nhwc(make_img(dy, N, C, H, W), g, s);
        norm_backward(xin, gamma, beta, act, g, o, rt.alloc_stats((size_t)N * C * 2), s);
        nhwc_to_nchw(o, dx, s);
    });
}

int tha4_test_tail_backward(tha4_ctx* ctx, int kind, const float* const* outputs, int N, int S, const float* image0,
                            const float* image1, const float* const* grad_outputs, float* d_head, float* d_image0,
                            float* d_image1, void* stream) {
    return guarded(ctx, [&] {
        cudaStream_t s = (cudaStream_t)stream;
        THA4_REQUIRE(kind >= TAIL_UNET && kind <= TAIL_FACE, "test_tail_backward: kind 0..3");
        THA4_REQUIRE(!image1 == (kind != TAIL_COMBINER), "test_tail_backward: image1 is the combiner's background layer");
        begin_pass(ctx, s);
        Pool* P = &ctx->persist;
        auto mk = [&](int c) { View v; v.N = N; v.H = S; v.W = S; v.C = c; v.ld = c; v.p = P->alloc((size_t)N * S * S * c); return v; };
        View dh = mk(16), dimg = mk(8);
        THA4_CUDA_CHECK(cudaMemsetAsync(dimg.p, 0, dimg.pixels() * 8 * sizeof(float), s));
        tail_backward((TailKind)kind, outputs, grad_outputs, make_img(image0, N, 4, S, S), image1 ? make_img(image1, N, 4, S, S) : ImgView{},
                      dh, d_image0 ? dimg.p : nullptr, d_image1 ? dimg.p + 4 : nullptr, 8, s);
        nhwc_to_nchw(dh.slice(0, 12), d_head, s);
        if (d_image0) nhwc_to_nchw(dimg.slice(0, 4), d_image0, s);
        if (d_image1) nhwc_to_nchw(dimg.slice(4, 4), d_image1, s);
    });
}

int tha4_test_upscaler_prologue_backward(tha4_ctx* ctx, const float* rest_image, const float* coarse_grid_change, int coarse_size,
                                         int N, const float* d_x0, float* d_rest_image, float* d_coarse_posed_image,
                                         float* d_coarse_grid_change, void* stream) {
    return guarded(ctx, [&] {
        cudaStream_t s = (cudaStream_t)stream;
        THA4_REQUIRE(coarse_size == 256 || coarse_size == 512, "test_upscaler_prologue_backward: coarse_size must be 256 or 512");
        begin_pass(ctx, s);
        Pool* P = &ctx->persist;
        auto mk = [&](int c) { View v; v.N = N; v.H = 512; v.W = 512; v.C = c; v.ld = c; v.p = P->alloc((size_t)N * 512 * 512 * c); return v; };
        View g = mk(16), dr = mk(4);
        nchw_to_nhwc(make_img(d_x0, N, 16, 512, 512), g, s);
        THA4_CUDA_CHECK(cudaMemsetAsync(dr.p, 0, dr.pixels() * 4 * sizeof(float), s));
        upscaler_prologue_backward(make_img(rest_image, N, 4, 512, 512), coarse_grid_change, coarse_size, g,
                                   d_rest_image ? dr.p : nullptr, d_coarse_posed_image, d_coarse_grid_change, s);
        if (d_rest_image) nhwc_to_nchw(dr, d_rest_image, s);
    });
}

int tha4_test_group_norm_backward(tha4_ctx* ctx, const float* x, int N, int C, int H, int W, int groups, const float* gamma,
                                  const float* beta, const float* film0, const float* film1, int act, const float* dy, float* dx,
                                  float* d_film, void* stream) {
    return guarded(ctx, [&] {
        cudaStream_t s = (cudaStream_t)stream;
        THA4_REQUIRE(act == ACT_NONE || act == ACT_SILU, "test_group_norm_backward: act 0 or 2");
        THA4_REQUIRE(!d_film || film1, "test_group_norm_backward: d_film needs film1");
        begin_pass(ctx, s);
        Runtime rt = make_rt(ctx, stream);
        Pool* P = &ctx->persist;
        auto mk = [&](int c) { View v; v.N = N; v.H = H; v.W = W; v.C = c; v.ld = c; v.p = P->alloc((size_t)N * H * W * c); return v; };
        View xin = mk(C);
        xin.stats_rep = 2; xin.stats_rep_stride = (long)N * C * 2;
        xin.stats = rt.alloc_stats((size_t)2 * N * C * 2); xin.stats_ld = C;
        nchw_to_nhwc(make_img(x, N, C, H, W), xin, s);
        norm_stats(xin, s);
        View g = mk(C), o = mk(C);
        nchw_to_nhwc(make_img(dy, N, C, H, W), g, s);
        group_norm_backward(xin, groups, gamma, beta, film0, film1, 2 * C, act, g, 0, o, d_film, 2 * C, nullptr, RES_NONE, nullptr,
                            rt.alloc_stats((size_t)N * C * 2), P->alloc((size_t)N * C * 8), s);
        nhwc_to_nchw(o, dx, s);
    });
}

int tha4_test_attention_backward(tha4_ctx* ctx, const float* qkv, const float* dout, int N, int C, int heads, float* dqkv, void* stream) {
    return guarded(ctx, [&] {
        cudaStream_t s = (cudaStream_t)stream;
        begin_pass(ctx, s);
        Pool* P = &ctx->persist;
        auto mk = [&](int c) { View v; v.N = N; v.H = 16; v.W = 16; v.C = c; v.ld = c; v.p = P->alloc((size_t)N * 256 * c); return v; };
        View q = mk(3 * C), g = mk(C), o = mk(3 * C);
        nchw_to_nhwc(make_img(qkv, N, 3 * C, 16, 16), q, s);
        nchw_to_nhwc(make_img(dout, N, C, 16, 16), g, s);
        attention_backward(q, g, heads, o, P->alloc((size_t)N * heads * 256 * 4), s);
        nhwc_to_nchw(o, dqkv, s);
    });
}

int tha4_test_attention(tha4_ctx* ctx, const float* qkv, int N, int C, int heads, float* out, void* stream) {
    return guarded(ctx, [&] {
        cudaStream_t s = (cudaStream_t)stream;
        begin_pass(ctx, (cudaStream_t)stream);
        Pool* P = &ctx->persist;
        View q; q.N = N; q.H = 16; q.W = 16; q.C = 3 * C; q.ld = 3 * C; q.p = P->alloc((size_t)N * 256 * 3 * C);
        nchw_to_nhwc(make_img(qkv, N, 3 * C, 16, 16), q, s);
        View o; o.N = N; o.H = 16; o.W = 16; o.C = C; o.ld = C; o.p = P->alloc((size_t)N * 256 * C);
        attention_forward(q, heads, o, s, !ctx->strict);
        nhwc_to_nchw(o, out, s);
    });
}

int tha4_test_linear(tha4_ctx* ctx, const float* x, int N, int I, const float* W, const float* b, int O, int silu_in,
                     float* y, void* stream) {
    return guarded(ctx, [&] { linear_forward(x, I, N, I, W, b, O, silu_in, y, O, (cudaStream_t)stream); });
}

int tha4_test_siren_level(tha4_ctx* ctx, int path, int mode, int n_tensors, const char* const* keys, const void* const* dev_ptrs,
                          const int64_t* shapes, const int* ndims, int n_layers, int has_head, int pose_dim, const int* npad,
                          const int* nb, const float* pose, int pose_ld, int B, const void* prev, int prev_c, const float* image,
                          int out_f16, void* const* outputs, void* stream) {
    return guarded(ctx, [&] {
        THA4_REQUIRE(path == 0 || path == 1, "siren level: path must be 0 (mma.sync) or 1 (wgmma)");
        begin_pass(ctx, (cudaStream_t)stream);
        Runtime rt = make_rt(ctx, stream);
        const StateDict sd = make_sd(n_tensors, keys, dev_ptrs, shapes, ndims);
        siren_test_level(rt, path == 1, mode, sd, n_layers, has_head != 0, pose_dim, npad, nb, pose, pose_ld, B,
                         (const __half*)prev, prev_c, image, out_f16 != 0, outputs);
    });
}

int tha4_test_sine(tha4_ctx* ctx, int which, const float* x, int64_t n, float* y, void* stream) {
    return guarded(ctx, [&] {
        THA4_REQUIRE(which == 0 || which == 1, "sine: which must be 0 (siren_sin) or 1 (st_sin)");
        if (which == 1) siren_tc_sine(x, (long)n, y, (cudaStream_t)stream);
        else siren_sine(x, (long)n, y, (cudaStream_t)stream);
    });
}

int tha4_test_siren_plan_check(int mode, int n_layers, const int* kpad, const int* npad, const int* nb, const int* sine,
                               const int* first, int R, int e_npad, int prev_c, int out_c, char* msg, int msg_len) {
    std::string err;
    if (n_layers < 0 || n_layers > 8 || (n_layers > 0 && (!kpad || !npad || !nb || !sine || !first))) {
        err = "layer count " + std::to_string(n_layers) + " is not 1..8";
    } else {
        SirenTcPlan plan;
        plan.nl = n_layers;
        for (int l = 0; l < n_layers; ++l) {
            plan.kpad[l] = kpad[l]; plan.npad[l] = npad[l]; plan.nb[l] = nb[l]; plan.sine[l] = sine[l]; plan.first[l] = first[l];
            plan.rows[l] = npad[l]; plan.W[l] = nullptr; plan.bias[l] = nullptr;
        }
        SirenTcLevel lv;
        lv.R = R; lv.e_npad = e_npad; lv.prev_c = prev_c; lv.out_c = out_c;
        err = siren_tc_plan_error(mode, plan, lv);
    }
    if (msg && msg_len > 0) {
        std::strncpy(msg, err.c_str(), (size_t)msg_len - 1);
        msg[msg_len - 1] = '\0';
    }
    return err.empty() ? THA4_OK : THA4_ERR_INVALID;
}

}  // extern "C"
