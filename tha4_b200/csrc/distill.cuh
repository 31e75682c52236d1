// Distillation inner loops of the body and face students (declarations) -- see distill.cu.
#pragma once
#include "nets.cuh"

namespace tha4 {

long siren_body_param_count();      // 331 567 (mode_14.py:108-131)

// One forward + backward of SirenMorpher03 on `image` ([N,4,512,512], the teacher's face_morphed_full) / `pose` against
// the teacher targets T0 (posed image), T2 (warped image), T3 (grid change).  loss_w: weights of the terms
// full_blended / full_warped / full_grid_change / full_color_change (siren_morpher_03_trainer.py:32-50).
// params / grads: flat fp32 buffers in state_dict order; grads is overwritten.  loss_acc: 4 doubles (device), the
// un-normalised sums of |a-b| of the four terms.
void siren_body_train_step(Runtime& rt, const ImgView& image, const float* pose, int pose_ld, const float* T0, const float* T2,
                           const float* T3, const float loss_w[4], const float* params, float* grads, double* loss_acc);

long siren_face_param_count();      // 121 476 (mode_14.py:93-105)

// One forward + backward of SirenFaceMorpher00 on `pose` ([N, >= 39], first 39 entries used) against `target`
// ([N,4,128,128]: the teacher's face crop) with the eye/mouth `mask` ([N,4,128,128]).  loss_w: weights of the plain and
// the masked L1 term (siren_face_morpher_00_trainer.py:168-186: 1.0 / 20.0).  loss_acc[0..1]: sums of |o-t| and |(t-o) m|.
void siren_face_train_step(Runtime& rt, const float* pose, int pose_ld, int N, const float* target, const float* mask,
                           const float loss_w[2], const float* params, float* grads, double* loss_acc);

// Largest batches of one train step / one backward micro-batch (the activation workspace scales with them).
constexpr int SIREN_BODY_MAX_BATCH = 8;
constexpr int SIREN_FACE_MAX_BATCH = 64;

// Parameter gradients of SirenMorpher03 for arbitrary upstream gradients (module-level autograd): forward with stored
// activations (TF32 products, as siren_body_train_step), then the backward from g[5] = d blended [N,4,512,512], d alpha
// [N,1,..], d color_change [N,4,..], d warped [N,4,..], d grid_change [N,2,..] (NCHW fp32; NULL = zero).  N <= 8.
// ACCUMULATES into grads: the caller zeroes it once for all micro-batches.
void siren_body_backward(Runtime& rt, const ImgView& image, const float* pose, int pose_ld, const float* const g[5], const float* params,
                         float* grads);
// Same for SirenFaceMorpher00: pose [N, >= 39] rows pose_ld apart, grad_output [N,4,128,128] NCHW.  N <= 64.
void siren_face_backward(Runtime& rt, const float* pose, int pose_ld, int N, const float* grad_output, const float* params, float* grads);

// torch.optim.Adam semantics on flat buffers; grads are multiplied by grad_scale first (1/world after an all-reduce sum).
void adam_step(float* params, const float* grads, float* m, float* v, long n, float lr, float beta1, float beta2, float eps,
               int step, float grad_scale, cudaStream_t s);

}  // namespace tha4
