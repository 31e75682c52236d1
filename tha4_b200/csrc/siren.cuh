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
};
void siren_tc_run(Runtime& rt, int mode, const SirenTcPlan& plan, const SirenTcLevel& lv);   // mode 0..2: body levels, 3: face
void siren_tc_enable(bool on);
bool siren_tc_enabled();

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

}  // namespace tha4
