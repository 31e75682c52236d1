/* tha4_b200 -- C ABI of the H100-native (sm_90a) THA4 poser hot path.
 *
 * The reference (pkhungurn/talking-head-anime-4-demo) is pure Python on PyTorch and has no FFI of its own
 * (SURVEY.md F1, section 8b): the seam it offers is Python duck-typing -- the `Poser` protocol
 * (src/tha4/poser/poser.py:132-161), `GeneralPoser02` (src/tha4/poser/general_poser_02.py:10-98) and the
 * `nn.Module.forward` signatures of the seven networks.  Each entry point below names the reference interface it
 * stands in for; the Python host mirror in tha4_b200/ binds them with ctypes (see INTEGRATION.md).
 *
 * Conventions: extern "C", no exceptions cross the boundary; every function returns 0 on success and a negative
 * code on failure, the message is available from tha4_last_error().  A context belongs to one (process, device)
 * and is NOT thread-safe.  All tensor arguments are raw device pointers to contiguous fp32 NCHW buffers owned by
 * the caller (e.g. torch tensors); `stream` is a cudaStream_t passed as void* (NULL = default stream).  The
 * library owns only its packed weights and its activation workspace.  There is no CPU fallback.
 */
#ifndef THA4_B200_H
#define THA4_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct tha4_ctx tha4_ctx;

#define THA4_OK 0
#define THA4_ERR_INVALID (-1)   /* bad argument / shape mismatch / missing weights */
#define THA4_ERR_CUDA (-2)      /* CUDA runtime error */

/* networks; the names are the keys of the reference's module dictionaries
 * (src/tha4/poser/modes/mode_07.py:20-25, src/tha4/poser/modes/mode_14.py:17-18) */
enum tha4_net {
    THA4_NET_EYEBROW_DECOMPOSER = 0,         /* EyebrowDecomposer00        */
    THA4_NET_EYEBROW_MORPHING_COMBINER = 1,  /* EyebrowMorphingCombiner00  */
    THA4_NET_FACE_MORPHER = 2,               /* FaceMorpher08              */
    THA4_NET_BODY_MORPHER = 3,               /* Morpher00                  */
    THA4_NET_UPSCALER = 4,                   /* Upscaler02                 */
    THA4_NET_SIREN_FACE_MORPHER = 5,         /* SirenFaceMorpher00         */
    THA4_NET_SIREN_BODY_MORPHER = 6,         /* SirenMorpher03             */
    THA4_NET_COUNT = 7
};

int tha4_ctx_create(int device, tha4_ctx** out);
int tha4_ctx_destroy(tha4_ctx* ctx);
/* message of the last failure on this context (ctx == NULL: last failure of context creation) */
const char* tha4_last_error(const tha4_ctx* ctx);

/* options: "strict" (0: tensor-core products on 10-bit-mantissa operands (f16 / TF32), fp32 accumulate -- the class of the
 *                       reference's own default on CUDA (cuDNN TF32 convs);
 *                    1: 3xTF32 error-compensated products == fp32 convolution; weights are re-uploaded on change;
 *                       teacher networks only -- the SIREN students always run fp16 operands / fp32 accumulate),
 *          "microbatch" (frames processed per pass of the teacher pipeline, default 32; bounds the workspace),
 *          "cuda_graphs" (default 1: a single-chunk teacher forward whose buffer set -- image, stream, output and cached
 *                         pointers -- repeats is captured once and replayed as one graph launch, writing the caller's
 *                         tensors directly; the pose is staged, so its address may change),
 *          developer switches, default = the measured-best setting:
 *          "tcgen05" (1: convs on the wgmma/TMA kernels; 0: everything on mma.sync; the name is historical),
 *          "half_operands" (1: f16 conv operands, normalisations fused into the consumer conv's operand path),
 *          "halo_conv" (1: 3x3 stride-1 convs on the halo-reuse kernel), "tma_store" (1: unsplit conv epilogue through TMA stores),
 *          "halo_m256" (-1: automatic; 0 / 1: force 128- / 256-pixel tiles on the unsplit launches of the halo kernel),
 *          "halo_ctas" (-1: automatic; 1 / 2: force one 288-thread / two 256-thread CTAs per SM for the halo kernel's
 *                       256 x 64 and four-phase tiles),
 *          "halo_cs" (-1: automatic; 1: never / 2: wherever legal split a one-CTA-per-SM launch of the halo kernel's 256 x 64 or
 *                     four-phase tiles over a cluster pair, each rank taking half of the channel chunks and finishing one
 *                     warpgroup's rows),
 *          "skip_fold" (1: the 1x1 skip of a U-Net ResBlock runs inside the K loop of the block's second conv, one halo launch;
 *                       0: its own launch on the side stream, added as conv1's residual),
 *          "cluster_splitk" (1: K-split convs reduce through a thread-block cluster / DSMEM; 0: workspace + reduce kernel),
 *          "siren_tc" (1: students on the wgmma kernels; 0: mma.sync kernels, one character only),
 *          "tail_persist" (1: persistent pipelined decoder tail; 0: one tile per CTA),
 *          "profile" (1: time every kernel class with CUDA events on the launching stream, 2: same + reset, 0: off).
 * Every option belongs to the context it is set on, except "profile": the profiler's accumulators, like the
 * "kernel_launches" counter, belong to the process, so profiling is on or off for all contexts.  Every change drops the
 * context's captured graphs.  A context is used by one thread at a time; the tensor-map caches shared between contexts
 * are mutex-protected. */
int tha4_set_option(tha4_ctx* ctx, const char* name, int64_t value);
/* counters: "kernel_launches" (kernels this library has launched so far, replayed graph nodes included), "workspace_bytes",
 *           "graph_replays" / "graph_captures" / "graph_failures",
 *           "prof_{us|launches|flops|bytes}_{conv|norm|tail|attn|glue|siren}" (profile mode; synchronises) */
int64_t tha4_get_counter(const tha4_ctx* ctx, const char* name);

/* Replaces module.load_state_dict(torch_load(file)) (src/tha4/poser/modes/mode_07.py:152-155 and siblings;
 * src/tha4/shion/core/load_save.py:12-14).  keys/dev_ptrs/shapes describe the reference-format state_dict with
 * the tensors already on the device (fp32, contiguous); shapes holds 4 int64 per tensor (trailing dims = 1).
 * The library packs what it needs into its own layouts; the caller's tensors may be freed afterwards. */
int tha4_load_net(tha4_ctx* ctx, int net, int n_tensors, const char* const* keys, const void* const* dev_ptrs,
                  const int64_t* shapes, const int* ndims, void* stream);

/* ---- module-level forwards (replace nn.Module.forward of the reference; output order = the INDEX_* constants) ---- */
/* EyebrowDecomposer00.forward (src/tha4/nn/eyebrow_decomposer/eyebrow_decomposer_00.py:46-64)
 * image [B,4,128,128] -> 6 outputs: eyebrow_layer(4) eyebrow_alpha(1) eyebrow_color(4) background_layer(4)
 * background_alpha(1) background_color(4) */
int tha4_eyebrow_decomposer_forward(tha4_ctx* ctx, const float* image, int B, float* const* outputs, void* stream);
/* EyebrowMorphingCombiner00.forward (src/tha4/nn/eyebrow_morphing_combiner/eyebrow_morphing_combiner_00.py:47-72)
 * background_layer, eyebrow_layer [B,4,128,128], pose [B,12] (row stride pose_ld) -> 8 outputs */
int tha4_eyebrow_morphing_combiner_forward(tha4_ctx* ctx, const float* background_layer, const float* eyebrow_layer,
                                           const float* pose, int pose_ld, int B, float* const* outputs, void* stream);
/* FaceMorpher08.forward (src/tha4/nn/face_morpher/face_morpher_08.py:158-193): image [B,4,192,192], pose [B,27] -> 8 */
int tha4_face_morpher_forward(tha4_ctx* ctx, const float* image, const float* pose, int pose_ld, int B,
                              float* const* outputs, void* stream);
/* Input gradients of the three encoder-decoder networks for upstream gradients of their outputs (grad_outputs: 6 / 8
 * entries in the forward's output order, NCHW, an entry may be NULL = zero).  Every gradient output is optional (NULL = not
 * computed), at least one must be non-NULL, and each is overwritten: d_image / d_background_layer / d_eyebrow_layer have the
 * shape of the input, d_pose is [B,12] / [B,27] (contiguous).  The forward is recomputed in the context's precision mode
 * (default: f16 operands; strict: 3xTF32) and differentiated with fp32 data gradients.  Any B >= 1 (micro-batched).
 * d_params: the parameter gradients summed over the batch, a flat fp32 buffer of tha4_net_param_count(net) floats holding
 * every state_dict tensor of the network in state_dict order (the order of the reference module's state_dict()), overwritten;
 * NULL = not computed.  It counts as an output, and one call computes it together with the input gradients. */
int tha4_eyebrow_decomposer_backward(tha4_ctx* ctx, const float* image, int B, const float* const* grad_outputs,
                                     float* d_image, float* d_params, void* stream);
int tha4_eyebrow_morphing_combiner_backward(tha4_ctx* ctx, const float* background_layer, const float* eyebrow_layer,
                                            const float* pose, int pose_ld, int B, const float* const* grad_outputs,
                                            float* d_background_layer, float* d_eyebrow_layer, float* d_pose, float* d_params,
                                            void* stream);
int tha4_face_morpher_backward(tha4_ctx* ctx, const float* image, const float* pose, int pose_ld, int B,
                               const float* const* grad_outputs, float* d_image, float* d_pose, float* d_params, void* stream);
/* Floats of the parameters of THA4_NET_EYEBROW_DECOMPOSER / _EYEBROW_MORPHING_COMBINER / _FACE_MORPHER / _BODY_MORPHER /
 * _UPSCALER (the length of the d_params of their backward entries); -1 for any other network. */
int64_t tha4_net_param_count(int net);
/* Morpher00.forward (src/tha4/nn/morpher/morpher_00.py:42-66): image [B,4,256,256], pose [B,6] ->
 * merged(4) alpha(1) warped(4) grid_change(2) direct(4) */
int tha4_morpher_forward(tha4_ctx* ctx, const float* image, const float* pose, int pose_ld, int B,
                         float* const* outputs, void* stream);
/* Input gradients of Morpher00 for upstream gradients of its 5 outputs (grad_outputs in the forward's output order, NCHW,
 * an entry may be NULL = zero), with the rules of the encoder-decoder entries above: d_image [B,4,256,256] and d_pose [B,6]
 * (contiguous) are optional (NULL = not computed), at least one non-NULL, each overwritten.  The forward is recomputed in the
 * context's precision mode and differentiated with fp32 data gradients.  Any B >= 1 (micro-batched).  The adjoint weights
 * are packed by the first call.  d_params: the parameter gradients, as for the encoder-decoder entries (34 682 119 floats,
 * state_dict order; the t = 0 time embedding and its FiLM projections included); NULL = not computed, counts as an output. */
int tha4_morpher_backward(tha4_ctx* ctx, const float* image, const float* pose, int pose_ld, int B,
                          const float* const* grad_outputs, float* d_image, float* d_pose, float* d_params, void* stream);
/* Upscaler02.forward (src/tha4/nn/upscaler/upscaler_02.py:59-96): rest_image [B,4,512,512], coarse_posed_image
 * [B,4,S,S], coarse_grid_change [B,2,S,S], pose [B,6] -> merged alpha warped grid_change direct.
 * coarse_size S = 512: the reference signature.  S = 256: the half-resolution body-morpher outputs; the bilinear x2
 * upsamples of the caller (src/tha4/poser/modes/mode_07.py:114-115) are then fused into the prologue kernel. */
int tha4_upscaler_forward(tha4_ctx* ctx, const float* rest_image, const float* coarse_posed_image,
                          const float* coarse_grid_change, int coarse_size, const float* pose, int pose_ld, int B,
                          float* const* outputs, void* stream);
/* Input gradients of Upscaler02 at the inputs of tha4_upscaler_forward (coarse_size 256 or 512) for upstream gradients of its
 * 5 outputs (grad_outputs in the forward's output order, NCHW, an entry may be NULL = zero), with the rules of
 * tha4_morpher_backward: d_rest_image [B,4,512,512], d_coarse_posed_image [B,4,S,S], d_coarse_grid_change [B,2,S,S] (S =
 * coarse_size; at 256 through the adjoint of the fused bilinear x2) and d_pose [B,6] (contiguous) are optional (NULL = not
 * computed), at least one non-NULL, each overwritten.  d_params: the parameter gradients, as for the encoder-decoder entries
 * (35 015 655 floats, state_dict order: the U-Net's tensors, then coarse_image_conv's; the t = 0 time embedding and its FiLM
 * projections included); NULL = not computed, counts as an output.  Any B >= 1, in passes of at most min(microbatch, 6)
 * frames (the backward's workspace is about 2.6 GiB per frame at 512x512), with d_params of at most min(microbatch, 4)
 * (the backward then also keeps every conv's operand: about 3.3 GiB per frame in strict mode).  The adjoint weights are
 * packed by the first call. */
int tha4_upscaler_backward(tha4_ctx* ctx, const float* rest_image, const float* coarse_posed_image, const float* coarse_grid_change,
                           int coarse_size, const float* pose, int pose_ld, int B, const float* const* grad_outputs,
                           float* d_rest_image, float* d_coarse_posed_image, float* d_coarse_grid_change, float* d_pose,
                           float* d_params, void* stream);
/* SirenFaceMorpher00.forward (src/tha4/nn/siren/face_morpher/siren_face_morpher_00.py:34-51): pose [B,39] -> [B,4,128,128] */
int tha4_siren_face_morpher_forward(tha4_ctx* ctx, const float* pose, int pose_ld, int B, float* output, void* stream);
/* SirenMorpher03.forward (src/tha4/nn/siren/morpher/siren_morpher_03.py:107-139): image [B,4,512,512], pose [B,45] ->
 * blended(4) alpha(1) color_change(4) warped(4) grid_change(2) */
int tha4_siren_morpher_forward(tha4_ctx* ctx, const float* image, const float* pose, int pose_ld, int B,
                               float* const* outputs, void* stream);

/* ---- poser-level forwards (replace GeneralPoser02.get_posing_outputs, general_poser_02.py:63-79) ---- */
/* mode 7: FiveStepPoserComputationProtocol (src/tha4/poser/modes/mode_07.py:47-134): 33 outputs in the order
 *   upscaler(5) face_morphed_full(1) body_morpher(5) face_morpher(8) eyebrow_morphing_combiner(8) eyebrow_decomposer(6)
 * mode 12: the face-only teacher (src/tha4/poser/modes/mode_12.py:41-96): 22 outputs, face(8) combiner(8) decomposer(6).
 * image [B,4,512,512], pose [B,45].  image_batch_stride: floats between consecutive images -- 4*512*512 for a dense
 * batch, 0 when ONE image is posed B times (what `image.expand(B, -1, -1, -1)` describes in PyTorch: a pose sweep
 * never materialises B copies).  cached_decomposer: NULL, or the 6 decomposer outputs of an earlier call with
 * the same image batch (the reference's eyebrow cache, mode_07.py:56-68); then the decomposer is skipped and the
 * last 6 entries of `outputs` are not written. */
int tha4_teacher_forward(tha4_ctx* ctx, int mode, const float* image, int64_t image_batch_stride, const float* pose, int B,
                         float* const* outputs, int eyebrow_morphed_image_index, const float* const* cached_decomposer, void* stream);
/* mode 14: TwoStepPoserComputationProtocol (src/tha4/poser/modes/mode_14.py:40-90): body(5) + face(1) */
int tha4_student_forward(tha4_ctx* ctx, const float* image, const float* pose, int B, float* const* outputs, void* stream);
/* same with a storage type for the image and the six outputs: io_dtype 0 = fp32 (identical to the call above), 1 = fp16
 * ("fp16 I/O + fp32 accumulate", BASELINE configs[2]: image [B,4,512,512] __half in, __half planes out; the pose stays
 * fp32).  The arithmetic is the same: fp16 operands, fp32 accumulation, results rounded once on the store. */
int tha4_student_forward_io(tha4_ctx* ctx, const void* image, const float* pose, int B, void* const* outputs, int io_dtype, void* stream);
/* ---- character bank: mode 14 for batches that mix characters ----
 * The reference deploys a student as a character model: one image plus one pair of student weight files
 * (src/tha4/charmodel/character_model.py:12-69), one poser per character.  A bank holds up to `capacity` character models
 * in one context, packed as tha4_load_net packs the two students but with the character as the outermost dimension of
 * every buffer, and tha4_bank_forward poses a batch in which every frame names its character: the wgmma student kernels
 * take a tile's weights, biases and image from the slot of the tile's frame.  A context has at most one bank;
 * tha4_bank_create replaces it, tha4_bank_destroy (and tha4_ctx_destroy) frees it. capacity: 1..4096; a character costs
 * about 0.9 MB of packed weights and 4 MB of image. */
int tha4_bank_create(tha4_ctx* ctx, int capacity);
int tha4_bank_destroy(tha4_ctx* ctx);
/* Fills (or replaces) slot 0 <= slot < capacity with one character: the state_dicts of SirenFaceMorpher00 and SirenMorpher03,
 * each described as for tha4_load_net, and its image [4,512,512] fp32 on the device (copied).  Other slots are not
 * touched.  Synchronises the device.  If the call fails the slot is left empty. */
int tha4_bank_set_character(tha4_ctx* ctx, int slot, int n_face, const char* const* face_keys, const void* const* face_ptrs,
                            const int64_t* face_shapes, const int* face_ndims, int n_body, const char* const* body_keys,
                            const void* const* body_ptrs, const int64_t* body_shapes, const int* body_ndims, const float* image,
                            void* stream);
/* tha4_student_forward_io for B frames of possibly different characters: frame n is the character in slot char_ids[n] at
 * pose[n] (pose [B,45] device fp32), its image is the slot's.  char_ids is a HOST array [B]: every id is checked
 * (0 <= id < capacity, slot filled) before anything is launched, then the library copies the array to the device itself.
 * outputs: the six of tha4_student_forward, fp32 (io_dtype 0) or fp16 (io_dtype 1; the slot's image is then rounded to
 * fp16 first, as the fp16 image of tha4_student_forward_io is).  A frame's outputs are bit-identical to what a context
 * holding that character alone returns for it.  wgmma kernels only: with option "siren_tc" = 0 the call is an error. */
int tha4_bank_forward(tha4_ctx* ctx, const int* char_ids, const float* pose, int B, void* const* outputs, int io_dtype, void* stream);
/* ---- distillation inner loop of the body student (replaces the autograd part of
 * SirenMorpherTrainingProtocol03.run_training_iteration, src/tha4/nn/siren/morpher/siren_morpher_protocols_03.py:178-214) ---- */
/* number of fp32 parameters of SirenMorpher03 in state_dict order (331 567) */
int64_t tha4_siren_morpher_param_count(void);
/* student forward + the four L1 terms (siren_morpher_03_trainer.py:32-50: blended vs target_posed, warped vs
 * target_warped, grid_change vs target_grid_change, color_change vs target_posed; mean reduction, weights
 * loss_weights[4] on the host) + full backward.  image = the teacher's face_morphed_full (output 5 of mode 7),
 * pose [B,45]; params / grads: flat device buffers in state_dict order (grads is overwritten);
 * host_loss_means (optional): the four unweighted means (synchronises).  B <= 8 per GPU as in the reference. */
int tha4_siren_morpher_train_step(tha4_ctx* ctx, const float* image, const float* pose, const float* target_posed,
                                  const float* target_warped, const float* target_grid_change, const float* loss_weights,
                                  const float* params, float* grads, double* host_loss_means, int B, void* stream);
/* Face student (SirenFaceMorpher00TrainerArgs, src/tha4/nn/siren/face_morpher/siren_face_morpher_00_trainer.py:101-186;
 * computation protocol siren_face_morpher_protocols_00.py:48-105): number of fp32 parameters in state_dict order (121 476) */
int64_t tha4_siren_face_morpher_param_count(void);
/* student forward on pose[:, 0:39] (pose rows pose_ld floats apart) + L1 against `target` [B,4,128,128] (the teacher's
 * mode-12 output 0 cropped as transform_poser_posed_image_to_groundtruth does, :123-126) + L1 of the difference
 * multiplied by `mask` [B,4,128,128] (MaskedL1Loss, shion/base/loss/l1_loss.py:40-58; eye_mouth_mask of the batch),
 * weights loss_weights[2] (1.0 / 20.0 in the reference), mean reduction + full backward.  params / grads as above.
 * host_loss_means (optional): the two unweighted means (synchronises). */
int tha4_siren_face_morpher_train_step(tha4_ctx* ctx, const float* pose, int pose_ld, const float* target, const float* mask,
                                       const float* loss_weights, const float* params, float* grads, double* host_loss_means,
                                       int B, void* stream);
/* ---- backward of the students under torch.autograd: parameter gradients, and input gradients of frozen students ---- */
/* ABI note: these two names used to declare parameter-gradient-only entries without the grid_change / alpha / d_image /
 * d_pose arguments.  A binding written against that signature must be updated; tha4_b200/_lib.py, the only one in this
 * tree, ships with the library.
 * The backward of SirenMorpher03 at (image [B,4,512,512], pose [B,45]) for upstream gradients grad_outputs[5] =
 * d blended, d alpha, d color_change, d warped, d grid_change (NCHW fp32, contiguous; NULL = zero).  Every output is
 * optional (NULL = not computed; at least one non-NULL; each is overwritten):
 *   grads   [331 567]      dL/d params, flat fp32 in state_dict order (params: the same layout).  The forward is
 *                          recomputed with TF32 products, as in tha4_siren_morpher_train_step;
 *   d_image [B,4,512,512]  dL/d image: the exact adjoint of the warp the forward returned, computed from its returned
 *                          grid_change [B,2,512,512] and alpha [B,1,512,512] and grad_outputs[0] / [3] (d blended,
 *                          d warped) with no SIREN recompute.  Float atomics: not bit-reproducible run to run;
 *   d_pose  [B,45]         dL/d pose of the TF32 recompute (as grads); fixed-order reduction, bit-reproducible.
 * grid_change / alpha are needed only for d_image; image / pose / params only for grads / d_pose.  Any B >= 1
 * (micro-batches of <= 8). */
int tha4_siren_morpher_backward(tha4_ctx* ctx, const float* image, const float* pose, int pose_ld, int B,
                                const float* const* grad_outputs, const float* grid_change, const float* alpha,
                                const float* params, float* grads, float* d_image, float* d_pose, void* stream);
/* The backward of SirenFaceMorpher00 at pose [B, >= 39] (rows pose_ld apart) for the upstream gradient grad_output
 * [B,4,128,128] (required), into grads [121 476] (as above) and / or d_pose [B,39] (every output optional, at least one
 * non-NULL, each overwritten).  Any B >= 1 (micro-batches of <= 64). */
int tha4_siren_face_morpher_backward(tha4_ctx* ctx, const float* pose, int pose_ld, int B, const float* grad_output,
                                     const float* params, float* grads, float* d_pose, void* stream);
/* torch.optim.Adam step on flat buffers (shion/base/optimizer_factories.py:9-17); grads are scaled by grad_scale first
 * (1/world_size after a summing all-reduce = DDP's gradient averaging) */
int tha4_adam_step(tha4_ctx* ctx, float* params, const float* grads, float* exp_avg, float* exp_avg_sq, int64_t n, float lr,
                   float beta1, float beta2, float eps, int step, float grad_scale, void* stream);

/* max|a-b| > 0 ?  -- the cache-validity test of mode_07.py:61 (synchronises the stream); result written to *differ */
int tha4_images_differ(tha4_ctx* ctx, const float* a, const float* b, int64_t n, int* differ, void* stream);

/* ---- image I/O on either side of the path (SURVEY 8f-1) ---- */
/* Poser output frame [B,4,H,W] fp32 in [-1,1] -> displayable [B,H,W,4] uint8 sRGB, the post-processing of the puppeteer
 * apps (src/tha4/app/character_model_ifacialmocap_puppeteer.py:325-349): clip((x+1)/2) -> linear->sRGB (RGB only) ->
 * background (0 none, 1 green, 2 blue, 3 black, 4 white: blend over it, alpha = 1) -> *255 -> uint8 (round_mode 0:
 * truncation as torch's .byte() there; 1: rint as tha4/image_util.py:56).  A 512x512 frame leaves the GPU as 1 MB. */
int tha4_frame_to_srgb8(tha4_ctx* ctx, const float* frame, int B, int H, int W, int background, int round_mode, uint8_t* out, void* stream);
/* PNG pixels [H,W,4] uint8 (sRGB, straight alpha) -> poser input [4,H,W] fp32 in [-1,1], linear RGB premultiplied by
 * alpha (src/tha4/shion/base/image_util.py:127-162) */
int tha4_rgba8_to_poser_image(tha4_ctx* ctx, const uint8_t* rgba, int H, int W, float* out, void* stream);

/* ---- kernel-level entry points (unit tests, ncu) ---- */
/* apply_grid_change (src/tha4/nn/image_processing_util.py:13-24): image [N,C,H,W], grid_change [N,2,H,W] ->
 * out [N,C,H,W]; optional corner indices x0,y0 [N,H,W] int32 and lerp weights tx,ty [N,H,W] (NULL to skip) */
int tha4_grid_sample(tha4_ctx* ctx, const float* image, const float* grid_change, int N, int C, int H, int W,
                     float* out, int32_t* x0, int32_t* y0, float* tx, float* ty, void* stream);
/* interpolate(mode='bilinear', align_corners=False) (mode_07.py:102,114-115) */
int tha4_resize_bilinear(tha4_ctx* ctx, const float* in, int N, int C, int Hi, int Wi, int Ho, int Wo, float* out, void* stream);
/* affine_grid(identity, align_corners=False) base coordinates for one axis (host output, `size` floats) */
int tha4_base_grid(int size, float* host_out);
/* conv kinds: 0 = 3x3 s1 p1, 1 = 4x4 s2 p1, 2 = transposed 4x4 s2 p1, 3 = 1x1, 4 = nearest x2 upsample + 3x3 s1 p1
 * (phase-decomposed on the low-resolution input).  x [N,Cin,H,W] (stored input; if
 * in_up the conv sees its nearest x2 upsample), w in the reference layout, bias / res may be NULL,
 * res_mode 1 same / 2 nearest-up x2 / 3 2x2 mean; y [N,Cout,Ho,Wo].  ksplit 0 = automatic. */
int tha4_test_conv(tha4_ctx* ctx, int kind, const float* x, const float* w, const float* bias, const float* res,
                   int res_mode, int in_up, float* y, int N, int Cin, int H, int W, int Cout, int strict, int ksplit,
                   void* stream);
/* conv(act(norm(x))) with the normalisation FUSED into the wgmma conv's operand path (default mode of the networks):
 * x [N,Cin,H,W] is the raw tensor; its first norm_C channels are normalised (groups 0: InstanceNorm2d, else GroupNorm;
 * FiLM vectors film0 [2*norm_C] / film1 [N,2*norm_C] optional; act 0 none / 1 relu / 2 silu), the remaining channels
 * pass through.  y: fp32 output [N,Cout,Ho,Wo]; y_from_f16 (optional): the f16 copy the kernel writes, widened. */
int tha4_test_conv_norm(tha4_ctx* ctx, int kind, const float* x, int N, int Cin, int H, int W, int norm_C, int groups,
                        const float* gamma, const float* beta, const float* film0, const float* film1, int act,
                        const float* w, const float* bias, const float* res, int res_mode, int Cout, int ksplit,
                        float* y, float* y_from_f16, void* stream);
/* same, and: norm_C = 0 convolves the raw input (no fused normalisation); y_stats (optional, device, [N,Cout,2] doubles): the
 * per-(n, c) sum and sum of squares of the fp32 output that the conv accumulates for its consumer's normalisation;
 * reps > 0: the conv is then launched `reps` more times between two CUDA events and *us_per_launch receives the mean
 * device time per launch (microseconds). */
int tha4_test_conv_norm_ex(tha4_ctx* ctx, int kind, const float* x, int N, int Cin, int H, int W, int norm_C, int groups,
                           const float* gamma, const float* beta, const float* film0, const float* film1, int act,
                           const float* w, const float* bias, const float* res, int res_mode, int Cout, int ksplit,
                           float* y, float* y_from_f16, double* y_stats, int reps, float* us_per_launch, void* stream);
/* y = act(norm(x)) with groups == 0: InstanceNorm2d, else GroupNorm(groups); act 0 none / 1 relu / 2 silu; pool 0/1;
 * film0 [2C] / film1 [N,2C] optional FiLM scale-shifts (unet.py:90-97); out_f16 = 1 runs the default-mode variant
 * (f16 output tensor, fast-math SiLU) and returns its values widened to fp32 */
/* The second conv of a U-Net ResBlock with a 1x1 skip: y = conv3x3(act(norm(x))) + bias + conv1x1(x2) + b_skip, x [N,Cmid,H,W]
 * the raw conv0 output (GroupNorm(groups) / InstanceNorm (groups 0) + film0 / film1 + act as in tha4_test_conv_norm_ex,
 * norm_C = Cmid), x2 [N,Cin2,H,W] the block input, w [Cout,Cmid,3,3], w_skip [Cout,Cin2,1,1].  With option "skip_fold" on,
 * one halo launch runs both (*folded = 1); with it off, the skip conv and conv1 with the skip as its residual (*folded = 0).  ksplit, y_stats, reps and us_per_launch as in tha4_test_conv_norm_ex (the
 * time is that of the one launch or of the pair). */
int tha4_test_conv_skip_fold(tha4_ctx* ctx, const float* x, int N, int Cmid, int H, int W, int groups, const float* gamma,
                             const float* beta, const float* film0, const float* film1, int act, const float* w, const float* bias,
                             const float* x2, int Cin2, const float* w_skip, const float* b_skip, int Cout, int ksplit,
                             float* y, double* y_stats, int* folded, int reps, float* us_per_launch, void* stream);
int tha4_test_norm(tha4_ctx* ctx, const float* x, int N, int C, int H, int W, int groups, const float* gamma,
                   const float* beta, const float* film0, const float* film1, int act, int pool, int out_f16, float* y, void* stream);
/* One fused decoder tail (SURVEY 8 a-T) in isolation: feature [N,C,S,S] is the raw last feature map; the kernel applies
 * the pending InstanceNorm (groups 0) / GroupNorm + activation (1 relu / 2 silu), the n_heads 3x3 head convs
 * (head_w: the reference weights [cout_i, C, 3, 3] concatenated in the order listed in tail.cu for `kind`, head_b:
 * concatenated biases incl. placeholders for bias-free heads), grid_sample and the blends.  kind 0 U-Net (5 outputs),
 * 1 decomposer (6), 2 combiner (8), 3 face morpher (8).  image1: combiner background layer, else NULL. */
int tha4_test_tail(tha4_ctx* ctx, int kind, const float* feature, int N, int C, int S, const float* gamma, const float* beta,
                   int groups, int act, const float* head_w, const float* head_b, const int* head_cout, int n_heads,
                   const float* image0, const float* image1, float* const* outputs, int strict, void* stream);
/* Data gradient of a conv on the conv kernels with adjoint-packed weights: kind 0 3x3 s1 p1 (w [Cout,Cin,3,3]), 1 4x4 s2 p1
 * (w [Cout,Cin,4,4]), 2 4x4 s2 p1 transposed (w [Cin,Cout,4,4]), 3 1x1 (w [Cout,Cin,1,1]), 4 nearest x2 upsample + 3x3 s1 p1
 * (w [Cout,Cin,3,3]; Ho = 2H), 5 3x3 s1 p1 as kind 0; dy [N,Cout,Ho,Wo] -> dx [N,Cin,H,W].  Cout % 4 == 0 (and Cin % 4 == 0
 * for kinds 1..4).  Kinds 3, 4 and 5 pack the forward conv first (Cin zero-padded to a multiple of 4, as the upscaler's fused
 * 16-channel first conv) and derive the adjoint from the packed weights, as the U-Net backward does.
 * strict: 3xTF32, else TF32 (fp32 operands in both). */
int tha4_test_conv_backward_data(tha4_ctx* ctx, int kind, const float* dy, const float* w, float* dx, int N, int Cin, int H, int W,
                                 int Cout, int strict, void* stream);
/* InstanceNorm2d(affine) (+ReLU when act == 1) backward: x, dy, dx [N,C,H,W] (statistics of x computed on the device) */
int tha4_test_norm_backward(tha4_ctx* ctx, const float* x, int N, int C, int H, int W, const float* gamma, const float* beta,
                            int act, const float* dy, float* dx, void* stream);
/* Tail backward of one kind (0 U-Net, 1 decomposer, 2 combiner, 3 face morpher) in isolation: outputs / grad_outputs as
 * tha4_test_tail returns them (grad entries may be NULL), image0 / image1 as for tha4_test_tail.  d_head [N,12,S,S]: gradients
 * of the head pre-activations in the channel order of tail.cu; d_image0 / d_image1 [N,4,S,S] (NULL = not computed). */
int tha4_test_tail_backward(tha4_ctx* ctx, int kind, const float* const* outputs, int N, int S, const float* image0,
                            const float* image1, const float* const* grad_outputs, float* d_head, float* d_image0,
                            float* d_image1, void* stream);
/* Adjoint of the Upscaler02 prologue (rest image, bilinear x2 of the coarse posed image and grid change, warp of the rest image
 * by the coarse grid; see tha4_upscaler_forward): rest_image [N,4,512,512], coarse_grid_change [N,2,S,S] (S = coarse_size,
 * 256 or 512), d_x0 [N,16,512,512] the gradient of the prologue's output channels rest(4) posed(4) warped(4) grid(2) pad(2)
 * -> d_rest_image [N,4,512,512], d_coarse_posed_image [N,4,S,S], d_coarse_grid_change [N,2,S,S] (NULL = not computed). */
int tha4_test_upscaler_prologue_backward(tha4_ctx* ctx, const float* rest_image, const float* coarse_grid_change, int coarse_size,
                                         int N, const float* d_x0, float* d_rest_image, float* d_coarse_posed_image,
                                         float* d_coarse_grid_change, void* stream);
/* GroupNorm(groups) (+FiLM) (+SiLU) backward of the U-Net ResBlocks (src/tha4/nn/common/unet.py:154-165): y = act(h), h =
 * (GN(x) * (1 + film0[c]) + film0[C+c]) * (1 + film1[n][c]) + film1[n][C+c] (film0 [2C], film1 [N,2C]; either may be NULL),
 * act 0 none / 2 SiLU.  x, dy, dx [N,C,H,W] (statistics of x computed on the device); d_film [N,2C] (NULL = not computed; needs
 * film1): d(scale) then d(shift) of film1.  C <= 512. */
int tha4_test_group_norm_backward(tha4_ctx* ctx, const float* x, int N, int C, int H, int W, int groups, const float* gamma,
                                  const float* beta, const float* film0, const float* film1, int act, const float* dy, float* dx,
                                  float* d_film, void* stream);
/* qkv_attention backward (fp32): qkv [N,3C,16,16], dout = d(attention output) [N,C,16,16] -> dqkv [N,3C,16,16] */
int tha4_test_attention_backward(tha4_ctx* ctx, const float* qkv, const float* dout, int N, int C, int heads, float* dqkv, void* stream);
/* The backward kernels in the layouts the network backwards run them.  Every tensor is an NHWC device tensor given by a
 * pointer to its channel 0 and a pixel stride (`*_ld`, in elements), so that it can be a channel slice of a wider buffer.
 * x (the raw input of the normalisation) is fp32, or f16 when x_f16; `stats` (device) holds its per-(n, c) sum and sum of
 * squares as stats_rep replicas [rep][N][stats_ld][2] (doubles), which the kernels add up.
 *
 * GroupNorm(groups) (+FiLM) (+SiLU) backward, group_norm_backward: film1 / d_film [N][film1_ld] / [N][d_film_ld] with this
 * layer's 2C columns at film1_off (d_film: d(scale) then d(shift); only those columns are written); dy [N,H,W,C], or
 * [N,H/2,W/2,C] when dy_pool (the output was 2x2-mean-pooled); res_mode 0 none, 1 same resolution, 2 the 2x2 sum of a
 * [N,2H,2W,C] res, 3 1/4 of a [N,H/2,W/2,C] res; add [N,H,W,C] or NULL.  C <= 512. */
int tha4_test_group_norm_backward_ex(tha4_ctx* ctx, const void* x, int x_f16, int x_ld, int N, int C, int H, int W, int groups,
                                     const double* stats, int stats_rep, int stats_ld, const float* gamma, const float* beta,
                                     const float* film0, const float* film1, int film1_ld, int film1_off, int act, const float* dy,
                                     int dy_ld, int dy_pool, const float* res, int res_ld, int res_mode, const float* add, int add_ld,
                                     float* dx, int dx_ld, float* d_film, int d_film_ld, void* stream);
/* The encoder-decoders' weight-gradient convolution (conv_wgrad.cu) through the launcher the network backward uses.  kind:
 * 0 3x3 s1 p1, 1 4x4 s2 p1, 2 transposed 4x4 s2 p1, 3 the heads' 3x3 with output channel d written at d * c_real * 9 (the
 * row map).  x: the forward conv's NHWC operand [N,H,W,x_ld] (f16 if x_f16), Cx channels; xf: 0 as stored, 1 the default
 * mode's fused InstanceNorm + ReLU (f16 coefficients from the statistics), 2 / 3 the tail's (fp32 affine; 3 rounds to f16)
 * on its first norm_C channels, statistics [stats_rep][N][norm_C][2].  dz: [N,Ho,Wo,dz_ld] fp32, Cout channels.  dW: the
 * reference layout ([Cout][c_real][k][k], transposed conv [Cx][Cout][4][4]; c_real 0 = every channel), written.
 * coef_out (optional): the [N][norm_C] (A, B) pairs the transform used.  plan[4]: N tile, M tiles, N tiles, pixel splits
 * (ksplit > 0 forces the split). */
int tha4_test_conv_wgrad(tha4_ctx* ctx, int kind, int strict, int ksplit, const void* x, int x_f16, int x_ld, int N, int H, int W,
                         int Cx, int xf, const double* stats, int stats_rep, const float* gamma, const float* beta, int norm_C,
                         const float* dz, int dz_ld, int Cout, int c_real, float* dW, float* coef_out, int* plan, void* stream);
/* The weight-gradient convolution's U-Net variants (Morpher00) through the same launcher.  kind: 0 3x3 s1 p1, 1 1x1, 2 nearest
 * x2 + 3x3 (x at half dz's resolution), 3 the last.2 head (3x3, Cout <= 16 channels in the N dimension).  x: [N,H,W,x_ld]
 * (f16 if x_f16), Cx channels; xf: 0 as stored, 1 the default mode's fused GroupNorm(groups) (+ FiLM0 [2 Cx] + FiLM1 row n
 * at film1 + film1_off, ld film1_ld) (+act) with f16 coefficients from the forward's builder, 2 / 3 the tail's (fp32 affine
 * from the statistics, 3 rounds to f16; no FiLM); act: 0 none, 1 ReLU, 2 SiLU, 3 the fast SiLU (tanh.approx) of the wgmma
 * kernels.  Statistics [stats_rep][N][Cx][2].  dz: [N,Ho,Wo,dz_ld] fp32, Cout channels.  dW: [Cout][Cx][k][k], written.
 * coef_out (optional): the [N][Cx] (A, B) pairs the transform used (f16 transform with SiLU: A / 2, B / 2).  plan[4]: as
 * tha4_test_conv_wgrad. */
int tha4_test_unet_wgrad(tha4_ctx* ctx, int kind, int strict, int ksplit, const void* x, int x_f16, int x_ld, int N, int H, int W,
                         int Cx, int xf, int act, const double* stats, int stats_rep, int groups, const float* gamma, const float* beta,
                         const float* film0, const float* film1, int film1_ld, int film1_off, const float* dz, int dz_ld, int Cout,
                         float* dW, float* coef_out, int* plan, void* stream);
/* InstanceNorm2d(affine) (+ReLU when act == 1) backward, norm_backward: x as above, dy / dx [N,H,W,C]. */
int tha4_test_norm_backward_ex(tha4_ctx* ctx, const void* x, int x_f16, int x_ld, int N, int C, int H, int W, const double* stats,
                               int stats_rep, int stats_ld, const float* gamma, const float* beta, int act, const float* dy, int dy_ld,
                               float* dx, int dx_ld, void* stream);
/* Conv data gradient through run_dgrad: kinds 0..5 and weights as tha4_test_conv_backward_data; kind 6 is the adjoint of the
 * fused tail's head conv from the 16-channel head gradient to Cin feature channels (Cout = 16; head_w / head_b / head_cout /
 * n_heads as for tha4_test_tail, packed with tail_init / tail_add and adjoint-packed by head_pack_adjoint).  dy
 * [N,Ho,Wo,Cout], dx [N,H,W,Cin rounded up to 4] (+ add of the same shape, or NULL).  workspace 0 runs the same conv without
 * the split-K workspace, so that a split launch that is not a cluster split accumulates atomically.  split_plan (host, may be
 * NULL) receives how the tensor-core kernel split K: 0 not split or not that kernel (strict mode), 1 cluster, 2 workspace,
 * 3 atomic. */
int tha4_test_conv_backward_data_ex(tha4_ctx* ctx, int kind, const float* w, const float* head_b, const int* head_cout, int n_heads,
                                    const float* dy, int dy_ld, const float* add, int add_ld, float* dx, int dx_ld, int N, int Cin,
                                    int H, int W, int Cout, int strict, int workspace, int* split_plan, void* stream);
/* linear_backward: dx[n][k] = SiLU'(pre[n][k]) sum_r dy[n][r] W[r][k] (pre NULL: no SiLU'), W [R][K] */
int tha4_test_linear_backward(tha4_ctx* ctx, const float* dy, int dy_ld, int N, int R, const float* W, int K, const float* pre, int pre_ld,
                              float* dx, int dx_ld, void* stream);
/* The parameter-gradient reductions of the network backwards, each through the launcher the networks call, on caller-owned
 * device buffers.  accumulate = 1 adds to the outputs instead of overwriting them.
 *
 * group_norm_backward as tha4_test_group_norm_backward_ex, then the GroupNorm (+FiLM) parameter fold of its per-(n, c) sums:
 * d_gamma / d_beta [C]; d_film0 (or NULL; needs film0): a row of d_film0_ld floats whose columns d_film0_off .. + 2C receive
 * d(scale0) then d(shift0), written whatever accumulate says; no other column is touched. */
int tha4_test_group_norm_param_grads(tha4_ctx* ctx, const void* x, int x_f16, int x_ld, int N, int C, int H, int W, int groups,
                                     const double* stats, int stats_rep, int stats_ld, const float* gamma, const float* beta,
                                     const float* film0, const float* film1, int film1_ld, int film1_off, int act, const float* dy,
                                     int dy_ld, int dy_pool, const float* res, int res_ld, int res_mode, const float* add, int add_ld,
                                     float* dx, int dx_ld, float* d_film, int d_film_ld, float* d_gamma, float* d_beta, float* d_film0,
                                     int d_film0_ld, int d_film0_off, int accumulate, void* stream);
/* norm_backward as tha4_test_norm_backward_ex, then the InstanceNorm parameter fold: d_gamma / d_beta [C]. */
int tha4_test_norm_param_grads(tha4_ctx* ctx, const void* x, int x_f16, int x_ld, int N, int C, int H, int W, const double* stats,
                               int stats_rep, int stats_ld, const float* gamma, const float* beta, int act, const float* dy, int dy_ld,
                               float* dx, int dx_ld, float* d_gamma, float* d_beta, int accumulate, void* stream);
/* Conv bias gradients: out[c] = sum over `pixels` rows of x [pixels][ld] of channel c < C; out2 (or NULL) gets the same. */
int tha4_test_channel_sums(tha4_ctx* ctx, const float* x, int ld, int64_t pixels, int C, float* out, float* out2, int accumulate,
                           void* stream);
/* Dense layer weight gradients: dW [R][K] = sum_n dy[n][r] u(x[n][k]), db [R] = sum_n dy[n][r], u = SiLU if silu_x. */
int tha4_test_linear_wgrad(tha4_ctx* ctx, const float* dy, int dy_ld, int N, int R, const float* x, int x_ld, int K, int silu_x,
                           float* dW, float* db, int accumulate, void* stream);
/* Encoder-decoder head biases: out[offsets[d]] = sum over the pixels of dh [pixels][16] of channel d < n <= 16; an offset
 * below 0 skips its channel. */
int tha4_test_head_bias(tha4_ctx* ctx, const float* dh, int64_t pixels, const int64_t* offsets, int n, float* out, int accumulate,
                        void* stream);
/* Encoder-decoder d(pose): dpose[n][k] = sum over the hw pixels of sample n < N of dbin [N][hw][ld] channel c0 + k, k < P. */
int tha4_test_pose_sum(tha4_ctx* ctx, const float* dbin, int ld, int64_t hw, int c0, int P, int N, float* dpose, int dpose_ld,
                       void* stream);
/* The default-mode forward kernels in the layouts the networks run them, on caller-owned device buffers so that a test can
 * chain launches into one concatenation buffer.  Tensors are NHWC, given by a pointer to their channel 0 and a pixel stride;
 * statistics slots by a pointer to their first column, a per-sample column stride stats_ld, `rep` replicas and the replica
 * stride in doubles ([rep][N][stats_ld][2] when the stride is N * stats_ld * 2).
 *
 * One conv through conv_forward: kind and weights (w [Cout,Cin,k,k], or [Cin,Cout,4,4] for kind 2; TF32-rounded and f16-packed
 * as the networks pack them) as tha4_test_conv; in [N,H,W,Cin] f16.  w_skip [Cout,Cin2,1,1] / b_skip / in2 [N,Ho,Wo,Cin2] f16:
 * a 1x1 skip folded into the 3x3 conv (conv_make_fold), or NULL.  out (fp32) and out16 (f16) are optional (at least one);
 * out_stats (or NULL) accumulates the output's per-(n, c) sums.  res fp32 with res_mode as tha4_test_conv (or NULL).  norm_C > 0:
 * the pending GroupNorm(groups) / InstanceNorm (groups 0) of the first norm_C input channels from in_stats, with gamma / beta,
 * film0 [2 norm_C] and film1 rows of film1_ld floats (or NULL), act 0 / 1 ReLU / 2 SiLU (run as the default mode's fast SiLU).
 * plan (host, 10 ints, may be NULL): [0] the kernel that ran (1 halo, 2 tensor-core, 3 mma.sync); for the halo kernel [1] N tile
 * [2] cluster size [3] consumer warpgroups [4] CTAs per SM [5] phases [6] TMA-store bits (1 fp32 out, 2 f16 out, 4 residual box)
 * [7] channel chunks [8] 1 when the skip was folded; [9] the tensor-core split plan (as tha4_test_conv_backward_data_ex). */
int tha4_test_conv_forward_ex(tha4_ctx* ctx, int kind, const float* w, const float* bias, int Cin, int Cout, const float* w_skip,
                              const float* b_skip, int Cin2, const void* in, int in_ld, int N, int H, int W, const void* in2, int in2_ld,
                              float* out, int out_ld, void* out16, int out16_ld, double* out_stats, int out_stats_ld, int out_stats_rep,
                              int64_t out_stats_rep_stride, const float* res, int res_ld, int res_mode, const double* in_stats,
                              int in_stats_ld, int in_stats_rep, int64_t in_stats_rep_stride, int norm_C, int groups, int act,
                              const float* gamma, const float* beta, const float* film0, const float* film1, int film1_ld, int ksplit,
                              int* plan, void* stream);
/* The default mode's fused tail (tail_tc_forward) on a raw f16 feature map [N,S,S,C] and its statistics replicas; heads,
 * gamma / beta / groups / act and outputs as tha4_test_tail.  image0 / image1 NCHW [.,4,S,S] with batch strides image*_sn
 * (0: one image for every sample); g0 / g1: their interleaved NHWC copies with pixel stride g*_ld (a slice of the network
 * input), or NULL (the kernel then reads the NCHW images). */
int tha4_test_tail_ex(tha4_ctx* ctx, int kind, const void* feature, int N, int C, int S, const double* stats, int stats_ld, int stats_rep,
                      int64_t stats_rep_stride, const float* gamma, const float* beta, int groups, int act, const float* head_w,
                      const float* head_b, const int* head_cout, int n_heads, const float* image0, int64_t image0_sn,
                      const float* image1, int64_t image1_sn, const float* g0, int g0_ld, const float* g1, int g1_ld,
                      float* const* outputs, void* stream);
/* qkv_attention, "new order" (src/tha4/nn/common/unet.py:192-202): qkv [N,3C,16,16] -> out [N,C,16,16] */
int tha4_test_attention(tha4_ctx* ctx, const float* qkv, int N, int C, int heads, float* out, void* stream);
/* y[n][o] = b[o] + sum_i f(x[n][i]) W[o][i] */
int tha4_test_linear(tha4_ctx* ctx, const float* x, int N, int I, const float* W, const float* b, int O, int silu_in,
                     float* y, void* stream);
/* One level of a SIREN student on path 1 (wgmma) or 0 (mma.sync).  mode 0..2: body levels 0..2 (R = 128, 256, 512),
 * 3: face (R = 128).  The layers come as a state_dict (described as for tha4_load_net) with the keys
 * "layer.<i>.weight" [N_i, Cin_i] / "layer.<i>.bias" [N_i] for i < n_layers, and "head.weight" / "head.bias" if has_head;
 * they are packed as the networks pack theirs.  Layer 0 is the level's first layer: its inputs are the previous level's
 * channels (modes 1 / 2), then x, y and the pose_dim pose entries.  npad[i]: the padded width of layer i (the next layer's
 * padded K); nb: the wgmma slice width of every GEMM layer in order, the head included (path 1; path 0 runs the production
 * shapes only).  pose [B, pose_ld]; prev: fp16 NHWC [B, R/2, R/2, prev_c] (modes 1 / 2); image [B,4,512,512] (level 2 with
 * a head).  outputs: without a head one fp16 NHWC tensor [B, R, R, npad[n_layers-1]]; level 2 with a head the five planes
 * blended(4) alpha(1) color(4) warped(4) grid_change(2), fp32 or (out_f16) fp16; the face with a head [B,4,128,128] fp32. */
int tha4_test_siren_level(tha4_ctx* ctx, int path, int mode, int n_tensors, const char* const* keys, const void* const* dev_ptrs,
                          const int64_t* shapes, const int* ndims, int n_layers, int has_head, int pose_dim, const int* npad,
                          const int* nb, const float* pose, int pose_ld, int B, const void* prev, int prev_c, const float* image,
                          int out_f16, void* const* outputs, void* stream);
/* y[i] = sin(x[i]) as the student kernels evaluate it: which 1 = the wgmma kernels' polynomial, 0 = the mma.sync kernels'
 * range reduction + __sinf */
int tha4_test_sine(tha4_ctx* ctx, int which, const float* x, int64_t n, float* y, void* stream);
/* ---- stages of the student training step (distill.cu), each through the host function the step calls ----
 * Tensors are device fp32, row-major [pixels][channels] (NHWC) as the step holds them. */
/* y [N*R*R][Cout] = x [N*R*R][Cin] W^T (+ bias_padded [Cout], may be NULL) on the wgmma 1x1 conv with W [nreal][kreal] packed
 * (TF32-rounded) by the step's packing kernel; transpose = 1: y = x W (Cin >= nreal, Cout >= kreal).  Channels past the real
 * ones are written as 0. */
int tha4_test_dense_gemm(tha4_ctx* ctx, const float* W, int nreal, int kreal, int transpose, const float* bias_padded, const float* x,
                         int Cin, float* y, int Cout, int N, int R, void* stream);
/* ACCUMULATES dW [nreal][kreal] += dz^T x and db [nreal] += column sums of dz over P pixels: dz [P][Nc], x [P][Kc] */
int tha4_test_dense_wgrad(tha4_ctx* ctx, const float* dz, int Nc, const float* x, int Kc, int64_t P, int nreal, int kreal, float* dW,
                          float* db, void* stream);
/* dir 0: the level input out [N][R][R][C] = [bilinear x2 of prev [N][R/2][R/2] (first Cprev of prev_ld channels) | x | y |
 * pose (npose of pose_ld per sample) | 0].  dir 1: its adjoint for the upsampled channels, out = dprev [N][R/2][R/2] (pixel
 * stride prev_ld; only channels 0..Cprev-1 are written) from up [N][R][R] (pixel stride up_ld). */
int tha4_test_level_input(tha4_ctx* ctx, int dir, const float* prev, int Cprev, int prev_ld, const float* pose, int pose_ld, int npose,
                          int R, int N, int C, const float* up, int up_ld, float* out, void* stream);
/* dir 0: out = sin(30 z); dir 1: out = da * 30 cos(30 z) (da is not modified).  n % 4 == 0. */
int tha4_test_distill_sine(tha4_ctx* ctx, int dir, const float* z, const float* da, int64_t n, float* out, void* stream);
/* d(pose) [N][npose] (overwritten) from 1..3 levels: level l has the first layer's dz [N][hw[l]][C[l]] and weight W[l]
 * [nreal[l]][kreal[l]] whose pose columns start at col0[l]. */
int tha4_test_pose_grad(tha4_ctx* ctx, int n_levels, const float* const* dz, const int* C, const int* hw, const float* const* W,
                        const int* nreal, const int* kreal, const int* col0, int N, int npose, float* dpose, void* stream);
/* Loss / gradient tails.  kind 0 (body loss): out = out7 [N*512*512][8], image [N,4,512,512], t0 / t1 / t2 = T0 posed / T2
 * warped [N,4,512,512], T3 grid change [N,2,512,512], loss_w[4]; loss_sums[4] (device doubles, overwritten) = the sums of |a-b|
 * of the four terms.  kind 1 (body upstream gradients): grads[5] = d blended, d alpha, d colour, d warped, d grid_change (NCHW,
 * entries or grads itself may be NULL = zero).  kind 2 (face loss): out = out4 [N*128*128][4], t0 = target, t1 = mask
 * [N,4,128,128], loss_w[2], loss_sums[0..1] (overwritten).  d_out: the gradient in the layout of out. */
int tha4_test_distill_tail(tha4_ctx* ctx, int kind, const float* out, const float* image, int N, const float* t0, const float* t1,
                           const float* t2, const float* const* grads, const float* loss_w, float* d_out, double* loss_sums, void* stream);
/* Host only, launches nothing: checks a wgmma student plan (per layer: padded K, padded N, slice width, sine 1 / head 0,
 * first-layer terms 0 / 1) for level `mode` with resolution R, elementwise first-layer width e_npad (modes 0 / 3), previous
 * level channels prev_c (modes 1 / 2) and output channels out_c.  Returns 0 if the kernel can run it, else
 * THA4_ERR_INVALID with the reason in msg (msg_len bytes, NUL-terminated). */
int tha4_test_siren_plan_check(int mode, int n_layers, const int* kpad, const int* npad, const int* nb, const int* sine,
                               const int* first, int R, int e_npad, int prev_c, int out_c, char* msg, int msg_len);

#ifdef __cplusplus
}
#endif
#endif /* THA4_B200_H */
