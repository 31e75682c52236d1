"""Developer script: A/B of one library option inside one process (device-resident B=1 teacher loop)."""
import os, sys, torch
_ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, _ROOT)
sys.path.insert(0, os.path.join(_ROOT, 'tests'))
from tha4_b200 import synthetic
from tha4_b200.poser.modes import mode_07
if len(sys.argv) != 2:
    sys.exit('usage: debug_ab.py OPTION   (an on/off option of tha4_set_option, e.g. skip_fold)')
opt = sys.argv[1]
dev = torch.device('cuda:0')
poser = mode_07.create_poser(dev, state_dicts=synthetic.teacher_state_dicts(0))
ctx = poser.get_context()
img = synthetic.synthetic_image(0, 1).to(dev); poses = synthetic.random_poses(64, seed=3).to(dev)
def run(n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for i in range(5): poser.get_posing_outputs(img, poses[i:i + 1])
    torch.cuda.synchronize(); e0.record()
    for i in range(n): poser.get_posing_outputs(img, poses[i % 64:i % 64 + 1])
    e1.record(); torch.cuda.synchronize()
    return n / e0.elapsed_time(e1) * 1e3
for v in (0, 1, 0, 1):
    ctx.set_option(opt, v)
    print(opt, v, round(run(40), 2), 'fps', flush=True)
