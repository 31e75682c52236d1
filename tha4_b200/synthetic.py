"""Seeded synthetic weights and inputs of the THA4 hot path (benchmarks, smoke tests, parity tests).

The teacher weights are not shipped with the reference (they are a separate download, README.md:164-183 there) and
657 MB of fp32 cannot be committed, so benchmarks and tests regenerate them from a seed with torch's CPU generator
(bit-identical across machines running the same torch build).  Tensors that the reference zero-initialises (U-Net
conv1 / last / attention out-proj, coarse_image_conv, grid_change heads) are drawn from small normals instead,
otherwise a random-init teacher outputs zero warps and nothing downstream is exercised.

Conditioning (round 2).  A plain He-init teacher is *chaotic* as a function of its conv operands: its heads paint
full-amplitude white noise, the next network warps that noise, and a 1e-3 change of a warp offset moves the result
by O(0.1) (scripts/dev/cpu_10bit_sensitivity.py: rounding the conv operands of the CPU oracle to 10 mantissa bits
moved the face-morpher outputs by 4.9e-2 mean).  Trained weights do not behave like that: residual branches are
small corrections, colour changes are small, alphas mostly keep the input image.  `_condition` gives the seeded
weights that character (key-name based scaling of the head / residual / zero-init tensors), which makes the fp32
oracle a usable yardstick for the tensor-core precision mode: the same 10-bit-operand emulation now moves every
mode_07 output by <= 3e-4 mean / 1.4e-2 max (scripts/dev/cpu_10bit_sensitivity.py, on the CPU), so the default-mode parity
tests can assert mean <= 2e-3, max <= 5e-2.
"""
import math
from typing import Dict

import torch

from tha4_b200.nn.state_dict_spec import Spec, STUDENT_SPECS, TEACHER_SPECS


def _draw(shape, role: str, g: torch.Generator) -> torch.Tensor:
    z = torch.randn(shape, generator=g, dtype=torch.float32)
    if role in ('conv', 'conv1'):
        fan_in = shape[1] * shape[2] * shape[3]
        return z * math.sqrt(2.0 / fan_in)
    if role == 'convT':      # kaiming_normal_ on [Cin, Cout, k, k]: torch's fan_in = size(1) * k * k
        return z * math.sqrt(2.0 / (shape[1] * shape[2] * shape[3]))
    if role == 'zconv':      # reference zero-inits; keep the residual branch at ~half scale
        return z * (0.5 * math.sqrt(1.0 / (shape[1] * shape[2] * shape[3])))
    if role == 'grid_head':  # reference zero-inits; warp offsets of ~0.05 in normalised coordinates
        return z * 0.003
    if role == 'last':       # reference zero-inits; direct ~0.4, grid ~0.04, alpha logit ~0.4
        w = z * (0.03 * math.sqrt(64.0 / shape[1]))
        w[4:6] *= 0.1
        return w
    if role == 'student_last':
        w = z * math.sqrt(2.0 / shape[1])
        w[0:2] *= 0.05
        return w
    if role == 'linear':
        return z * math.sqrt(1.0 / shape[1])
    if role == 'film':
        return z * (0.5 / math.sqrt(shape[1]))
    if role == 'norm_w':
        return 1.0 + 0.1 * z
    if role == 'norm_b':
        return 0.1 * z
    if role == 'bias':
        return 0.05 * z
    if role == 'siren_first':   # uniform(-1/in, 1/in) in the reference (siren.py:32); same scale here
        return (torch.rand(shape, generator=g) * 2 - 1) / shape[1]
    if role == 'siren':         # uniform(+-sqrt(6/in)/30) (siren.py:34-36)
        return (torch.rand(shape, generator=g) * 2 - 1) * (math.sqrt(6.0 / shape[1]) / 30.0)
    if role == 'siren_bias':
        return (torch.rand(shape, generator=g) * 2 - 1) * 0.05
    raise ValueError(role)


def _condition(key: str, shape, role: str, t: torch.Tensor) -> torch.Tensor:
    """Trained-like scaling of one seeded teacher tensor (see the module docstring)."""
    is_encdec_head = len(shape) == 4 and shape[1] == 64 and shape[2] == 3 and shape[0] <= 4 and not key.startswith('body.')
    if is_encdec_head and role == 'conv':
        return t * 0.1                                   # colour changes ~0.1, alpha logits ~ bias
    if role == 'bias' and 'alpha' in key and not key.startswith('body.'):
        # alphas keep the input image: eyebrow_layer = image * alpha + colour * (1 - alpha) wants alpha ~ 1,
        # every other blend is colour * alpha + image * (1 - alpha) and wants alpha ~ 0
        return t + (2.0 if key.startswith('eyebrow_layer_alpha') else -2.0)
    if role == 'grid_head':
        return t * 0.5                                   # warps of ~1-2 pixels
    if role == 'zconv':
        return t * 0.3                                   # residual branches are corrections, not replacements
    if role == 'last':
        return t * 0.3
    if key.endswith('resnet_path.4.weight'):             # InstanceNorm gamma that closes a ResnetBlock branch
        return t * 0.2
    if key == 'body.last.2.bias':
        t = t.clone()
        t[6] -= 2.0                                      # merged = direct * alpha + warped * (1 - alpha): mostly the warp
        return t
    return t


def make_state_dict(spec: Spec, seed: int, condition: bool = False) -> Dict[str, torch.Tensor]:
    g = torch.Generator().manual_seed(seed)
    out = {}
    for k, shape, role in spec:
        t = _draw(shape, role, g)
        out[k] = _condition(k, shape, role, t) if condition else t
    return out


def teacher_state_dicts(seed: int = 0) -> Dict[str, Dict[str, torch.Tensor]]:
    return {name: make_state_dict(fn(), seed * 100 + i, condition=True) for i, (name, fn) in enumerate(TEACHER_SPECS.items())}


def student_state_dicts(seed: int = 0) -> Dict[str, Dict[str, torch.Tensor]]:
    return {name: make_state_dict(fn(), seed * 100 + 50 + i) for i, (name, fn) in enumerate(STUDENT_SPECS.items())}


def synthetic_image(seed: int = 0, n: int = 1) -> torch.Tensor:
    """[n,4,512,512] in [-1,1]: smooth premultiplied-alpha-like blobs (not white noise, so that warps and
    bilinear taps see realistic gradients)."""
    g = torch.Generator().manual_seed(1000 + seed)
    low = torch.rand(n, 4, 32, 32, generator=g)
    img = torch.nn.functional.interpolate(low, size=(512, 512), mode='bicubic', align_corners=False).clamp(0, 1)
    img = img + 0.05 * torch.rand(n, 4, 512, 512, generator=g)
    alpha = img[:, 3:4].clamp(0, 1)
    img = torch.cat([img[:, 0:3].clamp(0, 1) * alpha, alpha], dim=1)
    return (img * 2.0 - 1.0).contiguous()


def random_poses(n: int, seed: int = 1234) -> torch.Tensor:
    """pose_i ~ U(range_i): morph parameters [0,1]; iris_rotation_x/y, head_x/y, neck_z, body_y/z in [-1,1];
    breathing [0,1]  (poser/modes/pose_parameters.py:6-35)."""
    g = torch.Generator().manual_seed(seed)
    u = torch.rand(n, 45, generator=g)
    lo = torch.zeros(45)
    lo[37:44] = -1.0
    return lo + u * (1.0 - lo)
