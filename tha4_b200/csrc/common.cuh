// Shared declarations for the tha4_b200 CUDA library (sm_90a: H100).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cstdint>
#include <cstdio>
#include <string>
#include <stdexcept>
#include <atomic>
#include <algorithm>
#include <vector>

namespace tha4 {

extern std::atomic<long> g_kernel_launches;   // every kernel this library launches is counted (bench "gpu_launches")

// The options of one context (tha4_set_option): its precision mode and which kernel and plan each launch takes.  Every API
// call binds its context's options to the calling thread for the duration of the call (OptionsScope), so the dispatchers
// read those of the context that is running; outside a call, opts() returns the defaults.
struct Options {
    bool strict = false;        // 3xTF32 error-compensated products (fp32-equivalent teacher convs) instead of TF32 / f16 operands
    int microbatch = 32;        // frames per internal pass of the teacher pipeline, 1..1024
    bool cuda_graphs = true;    // single-chunk teacher forwards on a repeating buffer set replay as one captured graph
    bool half_operands = true;  // f16 conv operands between a normalisation and the wgmma conv that reads it (non-strict mode)
    bool tcgen05 = true;        // convs on the wgmma / TMA kernels; off: every conv on mma.sync (the name is historical)
    bool cluster_splitk = true; // K-split wgmma convs reduce through a thread-block cluster; off: through a workspace or atomics
    bool halo_conv = true;      // 3x3 stride-1 and four-phase convs on the halo-reuse kernel; off: on conv_tc.cu
    bool tma_store = true;      // unsplit halo epilogues through shared-memory staging and TMA stores; off: plain stores
    int halo_m256 = -1;         // -1 automatic; 0 / 1 force 128- / 256-pixel tiles on unsplit halo launches
    int halo_ctas = -1;         // -1 automatic; 1 / 2 force one 288-thread / two 256-thread CTAs per SM (256 x 64 and four-phase tiles)
    int halo_cs = -1;           // -1 automatic; 1 never / 2 always (where legal) split a two-warpgroup halo launch over a cluster pair
    bool skip_fold = true;      // a U-Net ResBlock's 1x1 skip runs inside conv1's K loop (halo kernel); off: its own launch
    bool siren_tc = true;       // SIREN students on the wgmma kernels; off: on the mma.sync kernels (one character only)
    bool tail_persist = true;   // persistent pipelined wgmma decoder tail; off: one tile per CTA
};
extern thread_local const Options* g_options;
inline const Options& opts() {
    static const Options defaults;
    return g_options ? *g_options : defaults;
}
struct OptionsScope {
    const Options* prev;
    explicit OptionsScope(const Options* o) : prev(g_options) { g_options = o; }
    ~OptionsScope() { g_options = prev; }
};

// NHWC fp32 activation view.  `ld` is the pixel stride in floats (>= C) so that a tensor can live in a channel
// slice of a wider buffer (U-Net skip concatenation is free: producers write into their slice).
struct View {
    float* p = nullptr;
    int N = 0, H = 0, W = 0, C = 0, ld = 0;
    // f16 == 1: `p` really addresses __half elements (ld still counts elements).  Only the normalisation kernels write
    // such tensors and only the wgmma conv reads them (kind::f16 operands: same 10-bit mantissa as TF32, half the
    // operand bytes); everything else requires f16 == 0.
    int f16 = 0;
    // Optional per-(n,c) statistics of this tensor: stats[(n * stats_ld + c) * 2 + {0: sum, 1: sum of squares}] (doubles),
    // zero-initialised by the owner and accumulated by whichever kernel produces the tensor (conv epilogues).
    // Producers spread their atomics over `stats_rep` replicas (replica r at stats + r * stats_rep_stride) so that
    // thousands of tiles do not serialise on a handful of L2 lines; consumers add the replicas up.
    double* stats = nullptr;
    int stats_ld = 0;
    int stats_rep = 1;
    long stats_rep_stride = 0;
    __host__ __device__ long pix(int n, int y, int x) const { return (((long)n * H + y) * W + x) * ld; }
    View slice(int c0, int c) const {
        View v = *this;
        v.p = f16 ? reinterpret_cast<float*>(reinterpret_cast<__half*>(p) + c0) : p + c0;
        v.C = c; if (stats) v.stats = stats + 2 * c0; return v;
    }
    __half* hp() const { return reinterpret_cast<__half*>(p); }
    size_t pixels() const { return (size_t)N * H * W; }
};

// NCHW fp32 view with explicit strides (crops of a larger image need no copy).
struct ImgView {
    const float* p = nullptr;
    int N = 0, C = 0, H = 0, W = 0;
    long sn = 0, sc = 0, sh = 0;   // strides in floats; sw == 1
};
inline ImgView make_img(const float* p, int N, int C, int H, int W) {
    ImgView v; v.p = p; v.N = N; v.C = C; v.H = H; v.W = W; v.sc = (long)H * W; v.sn = (long)C * H * W; v.sh = W; return v;
}
inline ImgView crop_img(const ImgView& s, int y0, int x0, int h, int w) {
    ImgView v = s; v.p = s.p + (long)y0 * s.sh + x0; v.H = h; v.W = w; return v;
}

struct CudaError : std::runtime_error { using std::runtime_error::runtime_error; };

#define THA4_CUDA_CHECK(expr)                                                                     \
    do {                                                                                          \
        cudaError_t _e = (expr);                                                                  \
        if (_e != cudaSuccess)                                                                    \
            throw tha4::CudaError(std::string(#expr) + " failed: " + cudaGetErrorString(_e) +     \
                                  " at " + __FILE__ + ":" + std::to_string(__LINE__));            \
    } while (0)

#define THA4_LAUNCH_CHECK()                                                                       \
    do {                                                                                          \
        tha4::g_kernel_launches.fetch_add(1, std::memory_order_relaxed);                          \
        THA4_CUDA_CHECK(cudaGetLastError());                                                      \
    } while (0)

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) is a per-device property: every call site keeps what it has already
// configured per device (a process may hold contexts on several GPUs), not per process.
constexpr int THA4_MAX_DEVICES = 64;
inline int current_device() { int d = 0; cudaGetDevice(&d); return d < 0 || d >= THA4_MAX_DEVICES ? 0 : d; }
// streaming multiprocessors of the current device (132 on an H100 SXM): launch plans size their grids by it
inline int num_sms() {
    static int sms[THA4_MAX_DEVICES] = {};
    const int d = current_device();
    if (!sms[d]) { cudaDeviceGetAttribute(&sms[d], cudaDevAttrMultiProcessorCount, d); if (sms[d] <= 0) sms[d] = 132; }
    return sms[d];
}
#define THA4_ENSURE_SMEM(kernel, bytes)                                                           \
    do {                                                                                          \
        static size_t _cfg[tha4::THA4_MAX_DEVICES] = {};                                          \
        const int _d = tha4::current_device();                                                    \
        if (_cfg[_d] < (size_t)(bytes)) {                                                         \
            THA4_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(bytes))); \
            _cfg[_d] = (size_t)(bytes);                                                           \
        }                                                                                         \
    } while (0)

#define THA4_REQUIRE(cond, msg)                                                                   \
    do {                                                                                          \
        if (!(cond)) throw std::runtime_error(std::string("tha4: ") + (msg) + " [" #cond "] at " + \
                                              __FILE__ + ":" + std::to_string(__LINE__));         \
    } while (0)

// Programmatic dependent launch: a kernel launched through launch_pdl may start while its predecessor in the stream is
// still running; it must execute pdl_wait() before touching global memory (blocks until every earlier grid has
// completed and flushed) and should execute pdl_trigger() once it holds its resources (so that the NEXT kernel's
// prologue -- barrier init, descriptor prefetch, launch latency -- overlaps this one's body).
#ifdef __CUDACC__
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;\n" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;\n" ::: "memory"); }

template <typename... KArgs, typename... Args>
inline void launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, int cluster_z, Args&&... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = s;
    cudaLaunchAttribute attr[2];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    int na = 1;
    if (cluster_z > 1) {
        attr[na].id = cudaLaunchAttributeClusterDimension;
        attr[na].val.clusterDim.x = 1; attr[na].val.clusterDim.y = 1; attr[na].val.clusterDim.z = (unsigned)cluster_z;
        ++na;
    }
    cfg.attrs = attr; cfg.numAttrs = na;
    cudaError_t e = cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
    if (e != cudaSuccess)
        throw CudaError(std::string("cudaLaunchKernelEx failed: ") + cudaGetErrorString(e));
}
#endif

// Device allocations made while a network loads its weights are recorded in the network's AllocSink and released with
// it (weights are re-uploaded when the precision mode changes and after every distillation step).
struct AllocSink {
    std::vector<void*> ptrs;
    AllocSink() = default;
    AllocSink(const AllocSink&) = delete;
    AllocSink& operator=(const AllocSink&) = delete;
    ~AllocSink() { for (void* p : ptrs) cudaFree(p); }
};
extern thread_local AllocSink* g_alloc_sink;
struct SinkScope {
    AllocSink* prev;
    explicit SinkScope(AllocSink* s) : prev(g_alloc_sink) { g_alloc_sink = s; }
    ~SinkScope() { g_alloc_sink = prev; }
};
void* tracked_malloc(size_t bytes);      // cudaMalloc, recorded in the active sink (if any)

inline int ceil_div(long a, long b) { return (int)((a + b - 1) / b); }
inline int round_up(int a, int b) { return (a + b - 1) / b * b; }

enum Act { ACT_NONE = 0, ACT_RELU = 1, ACT_SILU = 2, ACT_SILU_FAST = 3 };   // FAST: ex2.approx / rcp.approx (default mode)

__device__ __forceinline__ float act_apply(float v, int act) {
    if (act == ACT_RELU) return fmaxf(v, 0.0f);
    if (act == ACT_SILU) return v / (1.0f + expf(-v));
    if (act == ACT_SILU_FAST) return __fdividef(v, 1.0f + __expf(-v));
    return v;
}
// round-to-nearest TF32 (10-bit mantissa) as the tensor cores would ideally see it; wgmma kind::tf32 truncates the
// low mantissa bits of what it reads, so producers of conv operands round once when they write (non-strict mode).
__device__ __forceinline__ float round_tf32(float v) {
    unsigned r;
    asm("cvt.rna.tf32.f32 %0, %1;\n" : "=r"(r) : "f"(v));
    return __uint_as_float(r);
}
__device__ __forceinline__ float sigmoid_f(float v) { return 1.0f / (1.0f + expf(-v)); }
// (sum, sum of squares) of one channel folded over the statistics replicas.  The loads are issued eight at a time before
// any of them is consumed: a dependent chain of up to 16 L2 round trips per channel was the single
// largest item in the prologue of every kernel that rebuilds a normalisation affine.
__device__ __forceinline__ double2 fold_stat_replicas(const double* __restrict__ p, long rep_stride, int rep) {
    double su = 0.0, sq = 0.0;
    for (int r0 = 0; r0 < rep; r0 += 8) {
        double2 v[8];
#pragma unroll
        for (int j = 0; j < 8; ++j)
            v[j] = (r0 + j < rep) ? __ldg(reinterpret_cast<const double2*>(p + (long)(r0 + j) * rep_stride)) : make_double2(0.0, 0.0);
#pragma unroll
        for (int j = 0; j < 8; ++j) { su += v[j].x; sq += v[j].y; }
    }
    return make_double2(su, sq);
}

// Same sum in the same order (replica 0 first), all loads of up to 16 replicas in flight at once: one L2 round trip.
__device__ __forceinline__ double2 fold_stat_replicas16(const double* __restrict__ p, long rep_stride, int rep) {
    if (rep > 16) return fold_stat_replicas(p, rep_stride, rep);
    double2 v[16];
#pragma unroll
    for (int j = 0; j < 16; ++j)
        v[j] = (j < rep) ? __ldg(reinterpret_cast<const double2*>(p + (long)j * rep_stride)) : make_double2(0.0, 0.0);
    double su = 0.0, sq = 0.0;
#pragma unroll
    for (int j = 0; j < 16; ++j) { su += v[j].x; sq += v[j].y; }
    return make_double2(su, sq);
}

}  // namespace tha4
