// SIREN student networks (declarations) -- see siren.cu.
#pragma once
#include "nets.cuh"

namespace tha4 {

struct SirenLayer {
    void* W = nullptr;        // __half [NPAD][KPAD], pre-scaled by omega_0
    float* bias = nullptr;    // [NPAD], pre-scaled
    float* wxy = nullptr;     // [NPAD][2]   (first layers only)
    float* wpose = nullptr;   // [NPAD][P]   (first layers only)
    int N = 0, NPAD = 0, KPAD = 0, P = 0;
    void load(const StateDict& sd, const std::string& prefix, int feat, int pose, int kpad, int npad, float scale, cudaStream_t s);
    // the packing of load() into buffers the caller owns (W / bias / wxy / wpose set, sized for kpad / npad / pose)
    void pack(const StateDict& sd, const std::string& prefix, int feat, int pose, int kpad, int npad, float scale, cudaStream_t s);
};

// ---- wgmma path (siren_tc.cu): a level = a chain of GEMM layers on 128-pixel tiles, weights streamed by TMA ----
struct SirenTcPlan {          // the GEMM layers of one kernel, in order
    int nl = 0;
    int kpad[8], npad[8], nb[8], sine[8], first[8], rows[8];
    const void* W[8]; const float* bias[8];
    void add(const SirenLayer& l, int nb, int sine, int first);
};
struct SirenTcLevel {
    int R = 0, B = 0;
    int e_npad = 0; const float* e_pb = nullptr; int e_pb_ld = 0; const float* e_wxy = nullptr;     // elementwise first layer (level 0, face)
    const float* f_pb = nullptr; int f_pb_ld = 0; const float* f_wxy = nullptr;                       // first GEMM layer of levels 1 / 2
    const __half* prev = nullptr; int prev_c = 0; __half* out = nullptr; int out_c = 0;
    ImgView image; float* o[5] = {nullptr, nullptr, nullptr, nullptr, nullptr}; bool o_f16 = false;
    float* face_out = nullptr; const float* head_bias = nullptr;
    // character bank: the plan's W / bias, e_wxy / f_wxy and head_bias point at character 0 of `chars` characters stored
    // back to back, and sample n runs on the weights of character char_of[n] (device, [B], every entry in 0..chars-1)
    const int* char_of = nullptr; int chars = 0; int head_cs = 0;     // head_cs: floats between two characters' head biases
};
void siren_tc_run(Runtime& rt, int mode, const SirenTcPlan& plan, const SirenTcLevel& lv);   // mode 0..2: body levels, 3: face
// Checks a plan against the kernel of `mode` (host only, launches nothing): "" if it fits, else what does not.  The
// kernel has no bounds checks of its own: K, N and the level's channel counts must fit its two operand buffers, its
// weight tiles and its first-layer staging area, or it reads and writes past them.  siren_tc_run calls it per launch.
std::string siren_tc_plan_error(int mode, const SirenTcPlan& plan, const SirenTcLevel& lv);
void siren_tc_sine(const float* x, long n, float* y, cudaStream_t s);     // y = st_sin(x) of the wgmma kernels
void siren_sine(const float* x, long n, float* y, cudaStream_t s);        // y = siren_sin(x) of the mma.sync kernels

// One level of a student network (mode 0..2: body levels 0..2, 3: face) on the wgmma path (tc) or the mma.sync path.
// L[0] is the level's first layer: its xy + pose columns enter through pb, the per-sample bias [B][L[0].NPAD], and
// L[0].wxy.  Modes 0 / 3 evaluate it elementwise; modes 1 / 2 run it as a GEMM on the bilinear x2 of `prev`.
// nb: the wgmma slice width of every GEMM layer in order, the head included.  Output: `out` [B,R,R,L[nl-1].NPAD] fp16
// NHWC without a head; the five tail planes (mode 2) or face_out [B,4,R,R] (mode 3) with one.
struct SirenLevelArgs {
    bool tc = true;
    int mode = 0, R = 0, B = 0;
    const SirenLayer* L = nullptr; int nl = 0; const SirenLayer* head = nullptr;
    const int* nb = nullptr;
    const float* pb = nullptr;
    const __half* prev = nullptr; int prev_c = 0;
    __half* out = nullptr;
    ImgView image; float* const* outputs = nullptr; bool out_f16 = false;
    float* face_out = nullptr;
    // character bank (wgmma path only): L / head are character 0 of `chars` characters whose buffers lie back to back
    // (SirenBank); sample n runs on character char_of[n] (device, [B]) and pb holds its per-sample bias
    const int* char_of = nullptr; int chars = 0;
};
void siren_level(Runtime& rt, const SirenLevelArgs& a);
// Kernel-level test entry: loads the layers "layer.<i>" (and "head") of `sd` as the networks do and runs one level.
void siren_test_level(Runtime& rt, bool tc, int mode, const StateDict& sd, int n_layers, bool has_head, int pose_dim,
                      const int* npad, const int* nb, const float* pose, int pose_ld, int B, const __half* prev, int prev_c,
                      const float* image, bool out_f16, void* const* outputs);

class SirenFaceNet {
public:
    void load(const StateDict& sd, cudaStream_t s);
    // pose: [B, >=39] with row stride pose_ld; out: [B,4,128,128] fp32 NCHW
    void forward(Runtime& rt, const float* pose, int pose_ld, int B, float* out);
    bool loaded() const { return loaded_; }
private:
    AllocSink owned_;
    SirenLayer layers_[8], head_;
    bool loaded_ = false;
};

class SirenBodyNet {
public:
    void load(const StateDict& sd, cudaStream_t s);
    // image: [B,4,512,512]; pose: [B,45]; outputs: blended(4) alpha(1) colour(4) warped(4) grid_change(2), fp32 NCHW
    // outputs_f16: the five output planes are __half (io_dtype = f16 of tha4_student_forward_io; wgmma path only)
    void forward(Runtime& rt, const ImgView& image, const float* pose, int pose_ld, float* const* outputs, bool outputs_f16 = false);
    bool loaded() const { return loaded_; }
private:
    AllocSink owned_;
    SirenLayer l_[3][3], head_;
    bool loaded_ = false;
};

// C characters' students in one set of buffers, for batches that mix characters (tha4_bank_forward).  Every layer is
// packed exactly as SirenFaceNet / SirenBodyNet pack it, into one allocation per layer with the character as the
// outermost dimension: W [C][NPAD][KPAD] fp16, bias [C][NPAD], wxy [C][NPAD][2], wpose [C][NPAD][P], head bias [C][8].
// The characters' images [C,4,512,512] fp32 live beside the weights, so a frame's image is addressed by its character.
class SirenBank {
public:
    explicit SirenBank(int capacity);
    int capacity() const { return capacity_; }
    bool filled(int slot) const { return slot >= 0 && slot < capacity_ && filled_[slot]; }
    // Packs one character into `slot` (other slots are not touched).  A slot whose packing fails is left empty.
    void set_character(int slot, const StateDict& face, const StateDict& body, const float* image, cudaStream_t s);
    // The mode_14 DAG for B frames: frame n is character char_of_host[n] (validated by the caller) at pose[n] ([B,45]).
    // outputs: the six of tha4_student_forward, fp32 or (outputs_f16) fp16; fp16 also rounds the image to fp16 first,
    // as the fp16 image of tha4_student_forward_io is.
    void forward(Runtime& rt, const int* char_of_host, const float* pose, int B, void* const* outputs, bool outputs_f16);
private:
    SirenLayer at(const SirenLayer& base, int slot) const;
    AllocSink owned_;
    int capacity_;
    std::vector<char> filled_;
    SirenLayer face_[8], face_head_, body_[3][3], body_head_;          // character 0; character c lies c layer sizes further
    float* images_ = nullptr;
};

}  // namespace tha4
