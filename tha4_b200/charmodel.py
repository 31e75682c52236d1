"""Many character models in one student batch.

The reference deploys the distilled student as a character model: one image plus one pair of student weight files
(src/tha4/charmodel/character_model.py:12-69), one `mode_14` poser per character.  A `CharacterBank` holds several of
them in one library context, and one call poses a batch in which every frame names its character (`tha4_bank_forward`:
the wgmma student kernels take a tile's weights, biases and image from the slot of the tile's frame).  A frame's outputs
are bit-identical to those of a `mode_14` poser that holds that character alone.

Inference only: calls run without autograd.  For gradients w.r.t. a pose or an image, compose the frozen student modules
as INTEGRATION.md section 2 shows.
"""
from typing import Dict, List, Optional, Sequence, Union

import torch
from torch import Tensor

from tha4_b200._lib import Context, Tha4Error
from tha4_b200.nn.state_dict_spec import STUDENT_SPECS

CharIds = Union[Sequence[int], Tensor]


def _check_state_dict(which: str, state_dict: Dict[str, Tensor]):
    spec = {k: shape for k, shape, _ in STUDENT_SPECS[which]()}
    missing = sorted(set(spec) - set(state_dict))
    unexpected = sorted(set(state_dict) - set(spec))
    if missing or unexpected:
        raise Tha4Error('%s state_dict does not have the student\'s keys: missing %s, unexpected %s' % (which, missing, unexpected))
    for k, shape in spec.items():
        if tuple(state_dict[k].shape) != shape:
            raise Tha4Error('%s state_dict: %s has shape %s, expected %s' % (which, k, tuple(state_dict[k].shape), shape))


class CharacterBank:
    def __init__(self, device: torch.device, capacity: int, context: Optional[Context] = None):
        """`capacity` empty character slots on `device`; `context`: an existing library context to put the bank on
        (a context holds one bank), default a context of its own."""
        if capacity < 1:
            raise Tha4Error('CharacterBank: capacity must be >= 1, got %d' % capacity)
        self._context = Context(device) if context is None else context
        self._device = self._context.device
        self._capacity = int(capacity)
        self._names: List[Optional[str]] = [None] * self._capacity
        self._context.bank_create(self._capacity)

    def get_context(self) -> Context:
        return self._context

    @property
    def capacity(self) -> int:
        return self._capacity

    @property
    def names(self) -> List[Optional[str]]:
        """The name in every slot (None: empty)."""
        return list(self._names)

    # ------------------------------------------------------------------ characters
    def add(self, name: str, image: Tensor, face_state_dict: Dict[str, Tensor], body_state_dict: Dict[str, Tensor]) -> int:
        """Puts a character into the first empty slot and returns the slot, which is its id in `pose`."""
        if None not in self._names:
            raise Tha4Error('CharacterBank: all %d slots are filled' % self._capacity)
        slot = self._names.index(None)
        self.replace(slot, name, image, face_state_dict, body_state_dict)
        return slot

    def replace(self, slot: int, name: str, image: Tensor, face_state_dict: Dict[str, Tensor],
                body_state_dict: Dict[str, Tensor]):
        """Fills `slot` with a character (image [4,512,512] as the posers take it); the other slots are not touched."""
        if not 0 <= slot < self._capacity:
            raise Tha4Error('CharacterBank: slot %d is not 0..%d' % (slot, self._capacity - 1))
        _check_state_dict('face_morpher', face_state_dict)
        _check_state_dict('body_morpher', body_state_dict)
        if tuple(image.shape) != (4, 512, 512):
            raise Tha4Error('CharacterBank: the image must be [4,512,512], got %s' % (tuple(image.shape),))
        self._names[slot] = None              # a failed upload leaves the slot empty
        self._context.bank_set_character(slot, face_state_dict, body_state_dict,
                                         image.detach().to(device=self._device, dtype=torch.float32))
        self._names[slot] = name

    # ------------------------------------------------------------------ posing
    def _ids(self, char_ids: CharIds) -> List[int]:
        if isinstance(char_ids, Tensor):
            if char_ids.dtype.is_floating_point or char_ids.dtype == torch.bool or char_ids.dim() != 1:
                raise Tha4Error('char_ids must be a one-dimensional integer tensor, got %s %s' % (char_ids.dtype, tuple(char_ids.shape)))
            char_ids = char_ids.tolist()
        ids = []
        for n, i in enumerate(char_ids):
            if isinstance(i, bool) or not isinstance(i, int):
                raise Tha4Error('char_ids[%d] = %r is not an integer' % (n, i))
            if not 0 <= i < self._capacity:
                raise Tha4Error('char_ids[%d] = %d is not a slot (0..%d)' % (n, i, self._capacity - 1))
            if self._names[i] is None:
                raise Tha4Error('char_ids[%d] = %d: the slot holds no character' % (n, i))
            ids.append(i)
        if not ids:
            raise Tha4Error('char_ids is empty')
        return ids

    def get_posing_outputs(self, char_ids: CharIds, poses: Tensor, half: bool = False) -> List[Tensor]:
        """The six `mode_14` outputs (body 5 + face 1) of frame n = character char_ids[n] at poses[n] ([B,45]).
        half: float16 outputs, as the `mode_14` poser returns for a float16 image."""
        if poses.requires_grad and torch.is_grad_enabled():
            raise Tha4Error('CharacterBank is inference only and poses requires grad: call it under torch.no_grad(), or '
                            'compose the frozen student modules for input gradients (INTEGRATION.md section 2)')
        ids = self._ids(char_ids)
        poses = poses.detach()
        poses = poses[None] if poses.dim() == 1 else poses
        if poses.shape != (len(ids), 45):
            raise Tha4Error('poses must be [%d,45] for %d character ids, got %s' % (len(ids), len(ids), tuple(poses.shape)))
        return self._context.bank_forward(ids, poses.float(), half)

    def pose(self, char_ids: CharIds, poses: Tensor, output_index: int = 0) -> Tensor:
        return self.get_posing_outputs(char_ids, poses)[output_index]

    def pose_to_srgb8(self, char_ids: CharIds, poses: Tensor, background=None, rint: bool = False, output_index: int = 0) -> Tensor:
        """`pose()` followed, on the GPU, by the display conversion of the puppeteer apps -> [B,512,512,4] uint8 sRGB."""
        return self._context.frame_to_srgb8(self.pose(char_ids, poses, output_index), background, rint)
