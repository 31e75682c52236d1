"""ctypes binding of libtha4_b200.so (include/tha4_b200.h) and the per-device Context wrapper.

PyTorch is used for device memory and streams only: tensors are allocated with torch and handed to the library as
raw pointers together with torch's current CUDA stream.
"""
import ctypes
import os
import weakref
from typing import Dict, List, Optional, Sequence

import torch
from torch import Tensor

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libtha4_b200.so')

NET_IDS = {
    'eyebrow_decomposer': 0, 'eyebrow_morphing_combiner': 1, 'face_morpher': 2, 'body_morpher': 3, 'upscaler': 4,
    'siren_face_morpher': 5, 'siren_body_morpher': 6,
}

# every symbol include/tha4_b200.h declares (tests check that the .so exports all of them)
EXPORTED_SYMBOLS = [
    'tha4_ctx_create', 'tha4_ctx_destroy', 'tha4_last_error', 'tha4_set_option', 'tha4_get_counter', 'tha4_load_net',
    'tha4_eyebrow_decomposer_forward', 'tha4_eyebrow_morphing_combiner_forward', 'tha4_face_morpher_forward',
    'tha4_morpher_forward', 'tha4_upscaler_forward', 'tha4_siren_face_morpher_forward', 'tha4_siren_morpher_forward',
    'tha4_teacher_forward', 'tha4_student_forward', 'tha4_student_forward_io', 'tha4_siren_morpher_param_count', 'tha4_siren_morpher_train_step',
    'tha4_siren_face_morpher_param_count', 'tha4_siren_face_morpher_train_step',
    'tha4_siren_morpher_backward', 'tha4_siren_face_morpher_backward',
    'tha4_adam_step', 'tha4_images_differ', 'tha4_frame_to_srgb8', 'tha4_rgba8_to_poser_image', 'tha4_grid_sample', 'tha4_resize_bilinear',
    'tha4_eyebrow_decomposer_backward', 'tha4_eyebrow_morphing_combiner_backward', 'tha4_face_morpher_backward',
    'tha4_morpher_backward', 'tha4_upscaler_backward',
    'tha4_test_conv_backward_data', 'tha4_test_norm_backward', 'tha4_test_tail_backward', 'tha4_test_upscaler_prologue_backward',
    'tha4_test_group_norm_backward', 'tha4_test_attention_backward',
    'tha4_base_grid', 'tha4_test_conv', 'tha4_test_conv_norm', 'tha4_test_conv_norm_ex', 'tha4_test_norm', 'tha4_test_tail', 'tha4_test_attention', 'tha4_test_linear',
    'tha4_test_siren_level', 'tha4_test_sine', 'tha4_test_siren_plan_check',
]

_lib = None


class Tha4Error(RuntimeError):
    pass


def load_library() -> ctypes.CDLL:
    """Loads libtha4_b200.so; raises (loudly) if it has not been built -- there is no fallback path."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise Tha4Error('tha4_b200: %s is missing -- build it with `python __graft_entry__.py` (nvcc, sm_100a). '
                        'There is no CPU / PyTorch fallback.' % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    lib.tha4_last_error.restype = ctypes.c_char_p
    lib.tha4_last_error.argtypes = [ctypes.c_void_p]
    lib.tha4_get_counter.restype = ctypes.c_int64
    lib.tha4_get_counter.argtypes = [ctypes.c_void_p, ctypes.c_char_p]
    lib.tha4_set_option.argtypes = [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_int64]
    lib.tha4_siren_morpher_param_count.restype = ctypes.c_int64
    lib.tha4_siren_face_morpher_param_count.restype = ctypes.c_int64
    lib.tha4_adam_step.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64,
                                   ctypes.c_float, ctypes.c_float, ctypes.c_float, ctypes.c_float, ctypes.c_int, ctypes.c_float,
                                   ctypes.c_void_p]
    lib.tha4_images_differ.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64,
                                       ctypes.POINTER(ctypes.c_int), ctypes.c_void_p]
    _lib = lib
    return lib


def _ptr(t: Optional[Tensor]):
    return ctypes.c_void_p(0 if t is None else t.data_ptr())


def _ptr_array(ts: Sequence[Optional[Tensor]]):
    return (ctypes.c_void_p * len(ts))(*[0 if t is None else t.data_ptr() for t in ts])


def _check_input(t: Tensor, device: torch.device, name: str) -> Tensor:
    if t.device != device:
        raise Tha4Error('%s is on %s but the poser lives on %s' % (name, t.device, device))
    if t.dtype != torch.float32:
        raise Tha4Error('%s must be float32 (Poser.get_dtype() == torch.float), got %s' % (name, t.dtype))
    return t.contiguous()


class Context:
    """One library context = one set of the seven networks + activation workspace on one CUDA device."""

    def __init__(self, device: torch.device):
        device = torch.device(device)
        if device.type != 'cuda':
            raise Tha4Error('tha4_b200 runs on CUDA devices only (no CPU fallback); got device %s' % device)
        if not torch.cuda.is_available():
            raise Tha4Error('tha4_b200: no CUDA device is available')
        self.device = torch.device('cuda', device.index if device.index is not None else torch.cuda.current_device())
        self.lib = load_library()
        handle = ctypes.c_void_p()
        rc = self.lib.tha4_ctx_create(self.device.index, ctypes.byref(handle))
        if rc != 0:
            raise Tha4Error('tha4_ctx_create failed: %s' % self.lib.tha4_last_error(None).decode())
        self.handle = handle
        self.loaded: Dict[str, object] = {}
        self.epoch = 0                       # bumped whenever options or weights change: results cached by callers are stale
        self.modules = weakref.WeakSet()     # NativeModules whose weights live in this context
        self.owners: Dict[str, object] = {}  # net name -> weakref to the module whose weights the library holds for it

    def __del__(self):
        try:
            if getattr(self, 'handle', None):
                self.lib.tha4_ctx_destroy(self.handle)
                self.handle = None
        except Exception:
            pass

    # ------------------------------------------------------------------ plumbing
    def _call(self, fn_name: str, *args):
        rc = getattr(self.lib, fn_name)(self.handle, *args)
        if rc != 0:
            raise Tha4Error('%s failed (%d): %s' % (fn_name, rc, self.lib.tha4_last_error(self.handle).decode()))

    def _stream(self):
        return ctypes.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def set_option(self, name: str, value: int):
        self._call('tha4_set_option', name.encode(), int(value))
        self.epoch += 1
        if name == 'strict':      # weight packing depends on it (TF32-rounded vs exact fp32): re-upload lazily
            for m in list(self.modules):
                m._uploaded_key = None

    def counter(self, name: str) -> int:
        return int(self.lib.tha4_get_counter(self.handle, name.encode()))

    def load_net(self, net: str, state_dict: Dict[str, Tensor]):
        """Hands a reference-format state_dict to the library (it packs its own copies)."""
        keys, tensors = [], []
        for k, v in state_dict.items():
            keys.append(k.encode())
            tensors.append(v.detach().to(device=self.device, dtype=torch.float32).contiguous())
        n = len(keys)
        shapes = (ctypes.c_int64 * (4 * n))()
        ndims = (ctypes.c_int * n)()
        for i, t in enumerate(tensors):
            ndims[i] = t.dim()
            for d in range(4):
                shapes[4 * i + d] = t.shape[d] if d < t.dim() else 1
        with torch.cuda.device(self.device):
            self._call('tha4_load_net', NET_IDS[net], n, (ctypes.c_char_p * n)(*keys), _ptr_array(tensors), shapes, ndims,
                       self._stream())
            torch.cuda.current_stream(self.device).synchronize()
        self.loaded[net] = True
        self.epoch += 1

    def _empty(self, specs, B: int) -> List[Tensor]:
        """Fresh output tensors for one call, carved out of ONE allocation (one allocator round trip instead of 33; and
        a loop that drops its previous outputs gets the same block -- hence the same addresses -- back from PyTorch's
        caching allocator, which is what lets the library replay a captured CUDA graph)."""
        sizes = [B * c * s * s for c, s in specs]
        offs, total = [], 0
        for n in sizes:
            offs.append(total)
            total += (n + 63) // 64 * 64                     # 256-byte aligned views (TMA / vector stores)
        flat = torch.empty((total,), dtype=torch.float32, device=self.device)
        return [flat[o:o + n].view(B, c, s, s) for o, n, (c, s) in zip(offs, sizes, specs)]

    # ------------------------------------------------------------------ module level
    def eyebrow_decomposer(self, image: Tensor) -> List[Tensor]:
        image = _check_input(image, self.device, 'image')
        assert image.shape[1:] == (4, 128, 128)
        B = image.shape[0]
        outs = self._empty([(4, 128), (1, 128), (4, 128), (4, 128), (1, 128), (4, 128)], B)
        self._call('tha4_eyebrow_decomposer_forward', _ptr(image), B, _ptr_array(outs), self._stream())
        return outs

    def eyebrow_morphing_combiner(self, background_layer: Tensor, eyebrow_layer: Tensor, pose: Tensor) -> List[Tensor]:
        background_layer = _check_input(background_layer, self.device, 'background_layer')
        eyebrow_layer = _check_input(eyebrow_layer, self.device, 'eyebrow_layer')
        pose = _check_input(pose, self.device, 'pose')
        B = background_layer.shape[0]
        assert background_layer.shape[1:] == (4, 128, 128) and eyebrow_layer.shape == background_layer.shape
        assert pose.shape == (B, 12)
        outs = self._empty([(4, 128), (1, 128), (4, 128), (4, 128), (1, 128), (4, 128), (4, 128), (2, 128)], B)
        self._call('tha4_eyebrow_morphing_combiner_forward', _ptr(background_layer), _ptr(eyebrow_layer), _ptr(pose), 12, B,
                   _ptr_array(outs), self._stream())
        return outs

    def face_morpher(self, image: Tensor, pose: Tensor) -> List[Tensor]:
        image = _check_input(image, self.device, 'image')
        pose = _check_input(pose, self.device, 'pose')
        B = image.shape[0]
        assert image.shape[1:] == (4, 192, 192) and pose.shape == (B, 27)
        outs = self._empty([(4, 192), (1, 192), (4, 192), (4, 192), (1, 192), (4, 192), (4, 192), (2, 192)], B)
        self._call('tha4_face_morpher_forward', _ptr(image), _ptr(pose), 27, B, _ptr_array(outs), self._stream())
        return outs

    DECOMPOSER_SPECS = [(4, 128), (1, 128), (4, 128), (4, 128), (1, 128), (4, 128)]
    COMBINER_SPECS = [(4, 128), (1, 128), (4, 128), (4, 128), (1, 128), (4, 128), (4, 128), (2, 128)]
    FACE_MORPHER_SPECS = [(4, 192), (1, 192), (4, 192), (4, 192), (1, 192), (4, 192), (4, 192), (2, 192)]

    def _grads(self, specs, grad_outputs: Sequence[Optional[Tensor]], B: int) -> List[Optional[Tensor]]:
        assert len(grad_outputs) == len(specs)
        gs = []
        for i, ((c, s), g) in enumerate(zip(specs, grad_outputs)):
            if g is not None:
                g = _check_input(g, self.device, 'gradient of output %d' % i)
                assert g.shape == (B, c, s, s), (i, tuple(g.shape))
            gs.append(g)
        return gs

    def eyebrow_decomposer_backward(self, image: Tensor, grad_outputs: Sequence[Optional[Tensor]], d_image: Tensor):
        """d_image [B,4,128,128] <- the input gradient of EyebrowDecomposer00 for the upstream gradients of its six outputs
        (None = zero); the forward is recomputed in the context's precision mode."""
        image = _check_input(image, self.device, 'image')
        B = image.shape[0]
        assert image.shape[1:] == (4, 128, 128)
        gs = self._grads(self.DECOMPOSER_SPECS, grad_outputs, B)
        self._check_out(d_image, (B, 4, 128, 128), 'd_image')
        self._call('tha4_eyebrow_decomposer_backward', _ptr(image), B, _ptr_array(gs), _ptr(d_image), self._stream())

    def eyebrow_morphing_combiner_backward(self, background_layer: Tensor, eyebrow_layer: Tensor, pose: Tensor,
                                           grad_outputs: Sequence[Optional[Tensor]], d_background_layer: Optional[Tensor] = None,
                                           d_eyebrow_layer: Optional[Tensor] = None, d_pose: Optional[Tensor] = None):
        """Input gradients of EyebrowMorphingCombiner00 into any of d_background_layer / d_eyebrow_layer [B,4,128,128] and
        d_pose [B,12] (None = not computed)."""
        assert d_background_layer is not None or d_eyebrow_layer is not None or d_pose is not None
        background_layer = _check_input(background_layer, self.device, 'background_layer')
        eyebrow_layer = _check_input(eyebrow_layer, self.device, 'eyebrow_layer')
        pose = _check_input(pose, self.device, 'pose')
        B = background_layer.shape[0]
        assert background_layer.shape[1:] == (4, 128, 128) and eyebrow_layer.shape == background_layer.shape and pose.shape == (B, 12)
        gs = self._grads(self.COMBINER_SPECS, grad_outputs, B)
        self._check_out(d_background_layer, (B, 4, 128, 128), 'd_background_layer')
        self._check_out(d_eyebrow_layer, (B, 4, 128, 128), 'd_eyebrow_layer')
        self._check_out(d_pose, (B, 12), 'd_pose')
        self._call('tha4_eyebrow_morphing_combiner_backward', _ptr(background_layer), _ptr(eyebrow_layer), _ptr(pose), 12, B,
                   _ptr_array(gs), _ptr(d_background_layer), _ptr(d_eyebrow_layer), _ptr(d_pose), self._stream())

    def face_morpher_backward(self, image: Tensor, pose: Tensor, grad_outputs: Sequence[Optional[Tensor]],
                              d_image: Optional[Tensor] = None, d_pose: Optional[Tensor] = None):
        """Input gradients of FaceMorpher08 into d_image [B,4,192,192] and / or d_pose [B,27] (None = not computed)."""
        assert d_image is not None or d_pose is not None
        image = _check_input(image, self.device, 'image')
        pose = _check_input(pose, self.device, 'pose')
        B = image.shape[0]
        assert image.shape[1:] == (4, 192, 192) and pose.shape == (B, 27)
        gs = self._grads(self.FACE_MORPHER_SPECS, grad_outputs, B)
        self._check_out(d_image, (B, 4, 192, 192), 'd_image')
        self._check_out(d_pose, (B, 27), 'd_pose')
        self._call('tha4_face_morpher_backward', _ptr(image), _ptr(pose), 27, B, _ptr_array(gs), _ptr(d_image), _ptr(d_pose),
                   self._stream())

    MORPHER_SPECS = [(4, 256), (1, 256), (4, 256), (2, 256), (4, 256)]

    def morpher(self, image: Tensor, pose: Tensor) -> List[Tensor]:
        image = _check_input(image, self.device, 'image')
        pose = _check_input(pose, self.device, 'pose')
        B = image.shape[0]
        outs = self._empty(self.MORPHER_SPECS, B)
        self._call('tha4_morpher_forward', _ptr(image), _ptr(pose), 6, B, _ptr_array(outs), self._stream())
        return outs

    def morpher_backward(self, image: Tensor, pose: Tensor, grad_outputs: Sequence[Optional[Tensor]],
                         d_image: Optional[Tensor] = None, d_pose: Optional[Tensor] = None):
        """Input gradients of Morpher00 into d_image [B,4,256,256] and / or d_pose [B,6] (None = not computed) for the upstream
        gradients of its five outputs (None = zero); the forward is recomputed in the context's precision mode."""
        assert d_image is not None or d_pose is not None
        image = _check_input(image, self.device, 'image')
        pose = _check_input(pose, self.device, 'pose')
        B = image.shape[0]
        assert image.shape[1:] == (4, 256, 256) and pose.shape == (B, 6)
        gs = self._grads(self.MORPHER_SPECS, grad_outputs, B)
        self._check_out(d_image, (B, 4, 256, 256), 'd_image')
        self._check_out(d_pose, (B, 6), 'd_pose')
        self._call('tha4_morpher_backward', _ptr(image), _ptr(pose), 6, B, _ptr_array(gs), _ptr(d_image), _ptr(d_pose),
                   self._stream())

    UPSCALER_SPECS = [(4, 512), (1, 512), (4, 512), (2, 512), (4, 512)]

    def _upscaler_inputs(self, rest_image: Tensor, coarse_posed: Tensor, coarse_grid: Tensor, pose: Tensor):
        rest_image = _check_input(rest_image, self.device, 'rest_image')
        coarse_posed = _check_input(coarse_posed, self.device, 'coarse_posed_image')
        coarse_grid = _check_input(coarse_grid, self.device, 'coarse_grid_change')
        pose = _check_input(pose, self.device, 'pose')
        B = rest_image.shape[0]
        S = coarse_posed.shape[2]
        assert rest_image.shape[1:] == (4, 512, 512) and S in (256, 512)
        assert coarse_posed.shape == (B, 4, S, S) and coarse_grid.shape == (B, 2, S, S) and pose.shape == (B, 6)
        return rest_image, coarse_posed, coarse_grid, pose, B, S

    def upscaler(self, rest_image: Tensor, coarse_posed: Tensor, coarse_grid: Tensor, pose: Tensor) -> List[Tensor]:
        rest_image, coarse_posed, coarse_grid, pose, B, S = self._upscaler_inputs(rest_image, coarse_posed, coarse_grid, pose)
        outs = self._empty(self.UPSCALER_SPECS, B)
        self._call('tha4_upscaler_forward', _ptr(rest_image), _ptr(coarse_posed), _ptr(coarse_grid), S, _ptr(pose), 6, B,
                   _ptr_array(outs), self._stream())
        return outs

    def upscaler_backward(self, rest_image: Tensor, coarse_posed: Tensor, coarse_grid: Tensor, pose: Tensor,
                          grad_outputs: Sequence[Optional[Tensor]], d_rest_image: Optional[Tensor] = None,
                          d_coarse_posed: Optional[Tensor] = None, d_coarse_grid: Optional[Tensor] = None,
                          d_pose: Optional[Tensor] = None):
        """Input gradients of Upscaler02 into any of d_rest_image [B,4,512,512], d_coarse_posed [B,4,S,S], d_coarse_grid
        [B,2,S,S] (S = the coarse inputs' size, 256 or 512) and d_pose [B,6] (None = not computed) for the upstream gradients
        of its five outputs (None = zero); the forward is recomputed in the context's precision mode."""
        assert d_rest_image is not None or d_coarse_posed is not None or d_coarse_grid is not None or d_pose is not None
        rest_image, coarse_posed, coarse_grid, pose, B, S = self._upscaler_inputs(rest_image, coarse_posed, coarse_grid, pose)
        gs = self._grads(self.UPSCALER_SPECS, grad_outputs, B)
        self._check_out(d_rest_image, (B, 4, 512, 512), 'd_rest_image')
        self._check_out(d_coarse_posed, (B, 4, S, S), 'd_coarse_posed')
        self._check_out(d_coarse_grid, (B, 2, S, S), 'd_coarse_grid')
        self._check_out(d_pose, (B, 6), 'd_pose')
        self._call('tha4_upscaler_backward', _ptr(rest_image), _ptr(coarse_posed), _ptr(coarse_grid), S, _ptr(pose), 6, B,
                   _ptr_array(gs), _ptr(d_rest_image), _ptr(d_coarse_posed), _ptr(d_coarse_grid), _ptr(d_pose), self._stream())

    def siren_face_morpher(self, pose: Tensor) -> Tensor:
        pose = _check_input(pose, self.device, 'pose')
        B = pose.shape[0]
        assert pose.shape == (B, 39)
        out = torch.empty((B, 4, 128, 128), dtype=torch.float32, device=self.device)
        self._call('tha4_siren_face_morpher_forward', _ptr(pose), 39, B, _ptr(out), self._stream())
        return out

    SIREN_MORPHER_SPECS = [(4, 512), (1, 512), (4, 512), (4, 512), (2, 512)]

    def siren_morpher(self, image: Tensor, pose: Tensor) -> List[Tensor]:
        B = image.shape[0]
        return self.siren_morpher_into(image, pose, self._empty(self.SIREN_MORPHER_SPECS, B))

    def siren_morpher_into(self, image: Tensor, pose: Tensor, outs: List[Tensor]) -> List[Tensor]:
        """SirenMorpher03 forward into caller-allocated contiguous outputs (shapes SIREN_MORPHER_SPECS)."""
        image = _check_input(image, self.device, 'image')
        pose = _check_input(pose, self.device, 'pose')
        B = image.shape[0]
        assert image.shape[1:] == (4, 512, 512) and pose.shape == (B, 45)
        for o, (c, s) in zip(outs, self.SIREN_MORPHER_SPECS):
            assert o.shape == (B, c, s, s) and o.is_contiguous() and o.dtype == torch.float32 and o.device == self.device
        self._call('tha4_siren_morpher_forward', _ptr(image), _ptr(pose), 45, B, _ptr_array(outs), self._stream())
        return outs

    # ------------------------------------------------------------------ poser level
    TEACHER_SPECS = {
        7: [(4, 512), (1, 512), (4, 512), (2, 512), (4, 512), (4, 512),
            (4, 256), (1, 256), (4, 256), (2, 256), (4, 256)],
        12: [],
    }
    FACE_COMB_DEC = [(4, 192), (1, 192), (4, 192), (4, 192), (1, 192), (4, 192), (4, 192), (2, 192),
                     (4, 128), (1, 128), (4, 128), (4, 128), (1, 128), (4, 128), (4, 128), (2, 128),
                     (4, 128), (1, 128), (4, 128), (4, 128), (1, 128), (4, 128)]

    def teacher_forward(self, mode: int, image: Tensor, pose: Tensor, eyebrow_morphed_image_index: int = 2,
                        cached_decomposer: Optional[List[Tensor]] = None) -> List[Tensor]:
        B = image.shape[0]
        if B > 1 and image.stride(0) == 0 and image[0].is_contiguous():
            # ONE image posed B times (image.expand(B, ...)): the library reads it with batch stride 0, no B-fold copy
            image0 = _check_input(image[0], self.device, 'image')
            img_ptr, img_stride, keep = _ptr(image0), 0, image0
        else:
            image = _check_input(image, self.device, 'image')
            img_ptr, img_stride, keep = _ptr(image), 4 * 512 * 512, image
        pose = _check_input(pose, self.device, 'pose')
        assert image.shape[1:] == (4, 512, 512) and pose.shape == (B, 45)
        specs = self.TEACHER_SPECS[mode] + self.FACE_COMB_DEC
        n = len(specs)
        if cached_decomposer is None:
            outs = self._empty(specs, B)
            cached = ctypes.c_void_p(0)
        else:
            outs = self._empty(specs[:n - 6], B) + list(cached_decomposer)
            cached = _ptr_array(cached_decomposer)
        self._call('tha4_teacher_forward', mode, img_ptr, ctypes.c_int64(img_stride), _ptr(pose), B, _ptr_array(outs),
                   eyebrow_morphed_image_index, cached, self._stream())
        del keep
        return outs

    def student_forward(self, image: Tensor, pose: Tensor) -> List[Tensor]:
        image = _check_input(image, self.device, 'image')
        pose = _check_input(pose, self.device, 'pose')
        B = image.shape[0]
        assert image.shape[1:] == (4, 512, 512) and pose.shape == (B, 45)
        outs = self._empty([(4, 512), (1, 512), (4, 512), (4, 512), (2, 512), (4, 128)], B)
        self._call('tha4_student_forward', _ptr(image), _ptr(pose), B, _ptr_array(outs), self._stream())
        return outs

    def student_forward_half(self, image: Tensor, pose: Tensor) -> List[Tensor]:
        """fp16 I/O variant (io_dtype = 1): half image in, half outputs out; the pose stays float32."""
        if image.device != self.device or image.dtype != torch.float16:
            raise Tha4Error('image must be a float16 tensor on %s' % self.device)
        image = image.contiguous()
        pose = _check_input(pose, self.device, 'pose')
        B = image.shape[0]
        assert image.shape[1:] == (4, 512, 512) and pose.shape == (B, 45)
        shapes = [(4, 512), (1, 512), (4, 512), (4, 512), (2, 512), (4, 128)]
        flat = torch.empty(sum(B * c * r * r for c, r in shapes), dtype=torch.float16, device=self.device)
        outs, o = [], 0
        for c, r in shapes:
            n = B * c * r * r
            outs.append(flat[o:o + n].view(B, c, r, r))
            o += n
        self._call('tha4_student_forward_io', _ptr(image), _ptr(pose), B, _ptr_array(outs), 1, self._stream())
        return outs

    # ------------------------------------------------------------------ distillation
    def siren_morpher_train_step(self, image: Tensor, pose: Tensor, target_posed: Tensor, target_warped: Tensor,
                                 target_grid_change: Tensor, loss_weights: Sequence[float], params: Tensor, grads: Tensor,
                                 want_losses: bool = True):
        tensors = [_check_input(t, self.device, n) for t, n in ((image, 'image'), (pose, 'pose'), (target_posed, 'target_posed'),
                                                                (target_warped, 'target_warped'), (target_grid_change, 'target_grid_change'))]
        B = image.shape[0]
        assert params.is_contiguous() and grads.is_contiguous() and params.dtype == torch.float32 and grads.dtype == torch.float32
        w = (ctypes.c_float * 4)(*[float(x) for x in loss_weights])
        losses = (ctypes.c_double * 4)()
        self._call('tha4_siren_morpher_train_step', *[_ptr(t) for t in tensors], w, _ptr(params), _ptr(grads),
                   losses if want_losses else None, B, self._stream())
        return list(losses) if want_losses else None

    def siren_face_morpher_train_step(self, pose: Tensor, target: Tensor, mask: Tensor, loss_weights: Sequence[float],
                                      params: Tensor, grads: Tensor, want_losses: bool = True):
        """pose [B, >= 39] (the first 39 entries are the student's input), target / mask [B,4,128,128]."""
        pose, target, mask = [_check_input(t, self.device, n) for t, n in ((pose, 'pose'), (target, 'target'), (mask, 'mask'))]
        B = pose.shape[0]
        assert target.shape == (B, 4, 128, 128) and mask.shape == (B, 4, 128, 128) and pose.shape[1] >= 39
        assert params.is_contiguous() and grads.is_contiguous() and params.dtype == torch.float32 and grads.dtype == torch.float32
        w = (ctypes.c_float * 2)(*[float(x) for x in loss_weights])
        losses = (ctypes.c_double * 2)()
        self._call('tha4_siren_face_morpher_train_step', _ptr(pose), int(pose.shape[1]), _ptr(target), _ptr(mask), w, _ptr(params),
                   _ptr(grads), losses if want_losses else None, B, self._stream())
        return list(losses) if want_losses else None

    @staticmethod
    def _check_out(t: Optional[Tensor], shape, name: str):
        if t is not None:
            assert t.shape == shape and t.is_contiguous() and t.dtype == torch.float32, (name, tuple(t.shape))

    @staticmethod
    def _check_flat(t: Optional[Tensor], n: int, name: str):
        """A flat fp32 buffer of a student's n parameters in state_dict order (params / grads)."""
        assert t is not None and t.is_contiguous() and t.dtype == torch.float32 and t.numel() == n, (name, n)

    def siren_morpher_backward(self, image: Tensor, pose: Tensor, grad_outputs: Sequence[Optional[Tensor]], *,
                               grid_change: Optional[Tensor] = None, alpha: Optional[Tensor] = None,
                               params: Optional[Tensor] = None, grads: Optional[Tensor] = None,
                               d_image: Optional[Tensor] = None, d_pose: Optional[Tensor] = None):
        """The backward of SirenMorpher03 for the upstream gradients of its five outputs (None = zero) into any of grads
        (dL/d params, flat in state_dict order), d_image [B,4,512,512] and d_pose [B,45] (None = not computed; the others
        are overwritten).  grads and d_pose recompute the forward with TF32 products, as the train step does, and need
        params; d_image is the adjoint of the warp the forward returned, from its grid_change / alpha outputs, with no
        SIREN recompute.  Any batch size."""
        assert grads is not None or d_image is not None or d_pose is not None
        image = _check_input(image, self.device, 'image')
        pose = _check_input(pose, self.device, 'pose')
        B = image.shape[0]
        assert image.shape[1:] == (4, 512, 512) and pose.shape == (B, 45)
        gs = self._grads(self.SIREN_MORPHER_SPECS, grad_outputs, B)
        if d_image is not None:
            assert grid_change is not None and alpha is not None, 'd_image needs the forward\'s grid_change and alpha'
            grid_change = _check_input(grid_change, self.device, 'grid_change')
            alpha = _check_input(alpha, self.device, 'alpha')
            assert grid_change.shape == (B, 2, 512, 512) and alpha.shape == (B, 1, 512, 512)
        n = self.lib.tha4_siren_morpher_param_count()
        if grads is not None or d_pose is not None:
            self._check_flat(params, n, 'params')
        if grads is not None:
            self._check_flat(grads, n, 'grads')
        self._check_out(d_image, (B, 4, 512, 512), 'd_image')
        self._check_out(d_pose, (B, 45), 'd_pose')
        self._call('tha4_siren_morpher_backward', _ptr(image), _ptr(pose), 45, B, _ptr_array(gs), _ptr(grid_change), _ptr(alpha),
                   _ptr(params), _ptr(grads), _ptr(d_image), _ptr(d_pose), self._stream())

    def siren_face_morpher_backward(self, pose: Tensor, grad_output: Tensor, params: Tensor, *, grads: Optional[Tensor] = None,
                                    d_pose: Optional[Tensor] = None):
        """The backward of SirenFaceMorpher00 for the upstream gradient [B,4,128,128] of its output into grads (dL/d params,
        flat in state_dict order) and / or d_pose [B,39] (None = not computed; the others are overwritten).  pose [B, >= 39]."""
        assert grads is not None or d_pose is not None
        pose = _check_input(pose, self.device, 'pose')
        grad_output = _check_input(grad_output, self.device, 'grad_output')
        B = pose.shape[0]
        assert pose.shape[1] >= 39 and grad_output.shape == (B, 4, 128, 128)
        n = self.lib.tha4_siren_face_morpher_param_count()
        self._check_flat(params, n, 'params')
        if grads is not None:
            self._check_flat(grads, n, 'grads')
        self._check_out(d_pose, (B, 39), 'd_pose')
        self._call('tha4_siren_face_morpher_backward', _ptr(pose), int(pose.shape[1]), B, _ptr(grad_output), _ptr(params),
                   _ptr(grads), _ptr(d_pose), self._stream())

    def adam_step(self, params: Tensor, grads: Tensor, exp_avg: Tensor, exp_avg_sq: Tensor, lr: float, step: int,
                  betas=(0.9, 0.999), eps: float = 1e-8, grad_scale: float = 1.0):
        rc = self.lib.tha4_adam_step(self.handle, _ptr(params), _ptr(grads), _ptr(exp_avg), _ptr(exp_avg_sq), params.numel(), lr,
                                     betas[0], betas[1], eps, step, grad_scale, self._stream())
        if rc != 0:
            raise Tha4Error('tha4_adam_step failed: %s' % self.lib.tha4_last_error(self.handle).decode())

    BACKGROUNDS = {None: 0, 'none': 0, 'green': 1, 'blue': 2, 'black': 3, 'white': 4}

    def frame_to_srgb8(self, frame: Tensor, background=None, rint: bool = False) -> Tensor:
        """[B,4,H,W] (or [4,H,W]) poser output -> [B,H,W,4] uint8 sRGB on the device (the puppeteers' display conversion)."""
        frame = _check_input(frame[None] if frame.dim() == 3 else frame, self.device, 'frame')
        B, C, H, W = frame.shape
        assert C == 4
        out = torch.empty((B, H, W, 4), dtype=torch.uint8, device=self.device)
        self._call('tha4_frame_to_srgb8', _ptr(frame), B, H, W, self.BACKGROUNDS[background], 1 if rint else 0, _ptr(out), self._stream())
        return out

    def rgba8_to_poser_image(self, rgba: Tensor) -> Tensor:
        """[H,W,4] uint8 PNG pixels on the device -> [4,H,W] fp32 poser input."""
        assert rgba.dtype == torch.uint8 and rgba.dim() == 3 and rgba.shape[2] == 4 and rgba.device == self.device
        rgba = rgba.contiguous()
        out = torch.empty((4, rgba.shape[0], rgba.shape[1]), dtype=torch.float32, device=self.device)
        self._call('tha4_rgba8_to_poser_image', _ptr(rgba), rgba.shape[0], rgba.shape[1], _ptr(out), self._stream())
        return out

    def images_differ(self, a: Tensor, b: Tensor) -> bool:
        a = _check_input(a, self.device, 'a')
        b = _check_input(b, self.device, 'b')
        flag = ctypes.c_int(0)
        self._call('tha4_images_differ', _ptr(a), _ptr(b), a.numel(), ctypes.byref(flag), self._stream())
        return flag.value != 0
