"""Developer timing of the character bank (not a pytest file), device time between CUDA events.

B = 64 student frames per step in every variant:
  one_character      Context.student_forward of lambda_00 at B = 64 (the workload `bench.py --workload student_b64` times)
  bank_C             one tha4_bank_forward of 64 frames drawn round-robin from C = 1, 2, 8, 64 bank slots (frame n is
                     character n mod C, so consecutive frames differ)
  contexts_C         C one-character contexts, each posing 64 / C frames per step: what a host without the bank runs
Slots beyond the two shipped characters hold seeded synthetic students.  Every variant is warmed first; then the variants
are timed alternately, `--repeats` rounds of at least `--seconds` of device work each, and the frames/s of every round is
printed so that the spread is visible.  Needs a GPU (no fallback).
Usage: python scripts/dev/bank_step.py [--seconds S] [--repeats R] [--max-characters C]"""
import argparse
import json
import os
import subprocess
import sys

import torch

_ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, _ROOT)
from tha4_b200 import image_util, synthetic  # noqa: E402
from tha4_b200._lib import Context  # noqa: E402
from tha4_b200.charmodel import CharacterBank  # noqa: E402

DEV = torch.device('cuda:0')
GOLDEN = os.path.join(_ROOT, 'tests', 'golden', 'data')
B = 64


def character(i):
    """(face state_dict, body state_dict, image [4,512,512]) of character i: 0 / 1 the shipped ones, then seeded students."""
    if i < 2:
        files = {'face_morpher': 'lambda_%02d_face_morpher.pt' % i,             # lambda_01's body weights are stored as fp16
                 'body_morpher': 'lambda_00_body_morpher.pt' if i == 0 else 'lambda_01_body_morpher_f16.pt'}
        sds = {k: {key: v.float() for key, v in torch.load(os.path.join(GOLDEN, f), map_location='cpu').items()} for k, f in files.items()}
        image = image_util.load_poser_image(os.path.join(GOLDEN, 'lambda_%02d.png' % i))
    else:
        sds = synthetic.student_state_dicts(i)
        image = synthetic.synthetic_image(i, 1)[0]
    return sds['face_morpher'], sds['body_morpher'], image


def one_context(i):
    face, body, image = character(i)
    ctx = Context(DEV)
    ctx.load_net('siren_face_morpher', face)
    ctx.load_net('siren_body_morpher', body)
    return ctx, image.to(DEV)


def device_seconds(fn, steps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e-3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--seconds', type=float, default=1.0, help='least device time of one timed round of one variant')
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--max-characters', type=int, default=64)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('bank_step.py: no CUDA device; the bank is timed on a GPU or not at all')
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                          capture_output=True, text=True, check=True).stdout.strip()
    print(json.dumps({'gpu': card, 'frames_per_step': B}), flush=True)

    counts = [c for c in (1, 2, 8, 64) if c <= args.max_characters]
    poses = synthetic.random_poses(B, seed=77).to(DEV)
    variants = {}

    contexts = [one_context(i) for i in range(max(counts))]
    ctx0, image0 = contexts[0]
    images0 = image0.unsqueeze(0).expand(B, -1, -1, -1).contiguous()
    variants['one_character'] = lambda: ctx0.student_forward(images0, poses)

    bank = CharacterBank(DEV, max(counts))
    for i in range(max(counts)):
        face, body, image = character(i)
        bank.add('character_%d' % i, image, face, body)
    for c in counts:
        ids = [n % c for n in range(B)]
        variants['bank_%d' % c] = lambda ids=ids: bank.get_posing_outputs(ids, poses)
    for c in counts:
        per = B // c
        batches = [(ctx, img.unsqueeze(0).expand(per, -1, -1, -1).contiguous(), poses[k * per:(k + 1) * per].contiguous())
                   for k, (ctx, img) in enumerate(contexts[:c])]
        variants['contexts_%d' % c] = lambda batches=batches: [ctx.student_forward(im, po) for ctx, im, po in batches]

    steps = {}
    for name, fn in variants.items():                  # warm every shape, and size the rounds
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        per_step = device_seconds(fn, 5) / 5
        steps[name] = max(5, int(args.seconds / per_step) + 1)
    rates = {name: [] for name in variants}
    for _ in range(args.repeats):
        for name, fn in variants.items():
            rates[name].append(B * steps[name] / device_seconds(fn, steps[name]))
    for name in variants:
        r = rates[name]
        print(json.dumps({'variant': name, 'steps_per_round': steps[name], 'frames_per_s': [round(x, 1) for x in r],
                          'min': round(min(r), 1), 'max': round(max(r), 1)}), flush=True)


if __name__ == '__main__':
    main()
