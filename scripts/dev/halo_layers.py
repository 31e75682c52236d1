"""Developer measurement of the 3x3 halo convolution in the teacher_b1 frame (not a pytest file).

1. The card's name and power limit.
2. One warm teacher_b1 frame (mode_07, batch 1, eyebrow cache hot) under torch.profiler with CUDA activities, with
   128-pixel halo tiles forced (option halo_m256 = 0), with one CTA per SM forced for the 256 x 64 and four-phase tiles
   (halo_ctas = 1), and with the automatic choice: device time per kernel instantiation, and the share of the unsplit
   halo launches; the same with no cluster pairs (halo_cs = 1).  Then every halo launch of the automatic frame with fewer CTAs than SMs (the launch log zipped with the
   trace's halo kernels) and their summed device time.
3. Every unsplit 3x3 halo conv shape of that frame (read from the library's launch log, THA4_HALO_DEBUG=2, in a child
   process) timed alone with CUDA events over --reps launches after warm-up, with 128- and with 256-pixel tiles:
   microseconds, TFLOP/s, and the compulsory HBM bytes computed from the shape (f16 input, f16 weights, the fp32 and f16
   outputs, the fp32 residual).  The 256-pixel tiles run with one and with two CTAs per SM (halo_ctas = 1 / 2; the
   same kernel where the tile is not 256 x 64), and on a row-owning cluster pair (halo_cs = 2: each rank half of the channel
   chunks, one warpgroup's rows).  The conv runs through the kernel-level test hook with the frame's input-normalisation
   kind and residual; the hook always writes both outputs.
4. Every four-phase shape of the teacher frame (nearest-x2 + 3x3 of the up-sampling ResBlocks, transposed 4x4 convs),
   and two at batch 32, timed the same way on three paths: conv_tc.cu's automatic plan (halo_conv = 0), the four-phase
   halo kernel (halo_conv = 1, an unsplit launch requested) with one and with two CTAs per SM (halo_ctas = 1 / 2), on a
   row-owning cluster pair (halo_cs = 2), and
   the automatic choice; TFLOP/s count the executed products (4 phases x 4 taps per low-resolution pixel).

Usage: python scripts/dev/halo_layers.py [--reps 200] [--out DIR] [--phase-only]
"""
import argparse
import collections
import os
import re
import subprocess
import sys

import torch

_ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, _ROOT)
sys.path.insert(0, os.path.join(_ROOT, 'tests'))

LAUNCH_RE = re.compile(r'halo launch: N (\d+) (\d+)x(\d+) cin (\d+) cout (\d+) \| bn (\d+) cs (\d+) wg (\d+) chunks (\d+) grid (\d+) x (\d+) \| '
                       r'xf (\d+) groups (\d+) act (\d+) res (\d+) out32 (\d+) out16 (\d+) st_tma (\d+) \| phases (\d+) ctas (\d+)')


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        q = 'nvidia-smi unavailable (%s)' % e
    return '%s | power limit, max SM clock: %s' % (name, q)


def make_teacher():
    import bench
    from tha4_b200 import synthetic
    from tha4_b200.poser.modes import mode_07
    device = torch.device('cuda:0')
    tsds, _ = bench.load_state_dicts('mode_07')
    poser = mode_07.create_poser(device, state_dicts=tsds)
    poser.get_modules()
    poser.protocol.trust_image_identity = True
    image = bench.load_image().to(device).unsqueeze(0).contiguous()
    poses = synthetic.random_poses(8, seed=1234).to(device)
    return poser, image, poses


def frame_shapes():
    """Runs two frames in a child process with the launch log on; returns the halo launches of the second (eyebrow cache
    hot) frame as dicts, in frame order."""
    code = ('import sys; sys.path.insert(0, %r); sys.path.insert(0, %r); import torch\n'
            'from halo_layers import make_teacher\n'
            'p, img, poses = make_teacher()\n'
            'with torch.no_grad():\n'
            '    p.get_posing_outputs(img, poses[0:1]); torch.cuda.synchronize()\n'
            '    sys.stderr.write("SECOND FRAME\\n"); sys.stderr.flush()\n'
            '    p.get_posing_outputs(img, poses[1:2]); torch.cuda.synchronize()\n') % (_ROOT, os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, THA4_HALO_DEBUG='2')
    r = subprocess.run([sys.executable, '-c', code], capture_output=True, text=True, env=env, cwd=_ROOT)
    if r.returncode != 0:
        raise RuntimeError('launch-log run failed:\n' + r.stderr[-4000:])
    keys = ('N', 'H', 'W', 'cin', 'cout', 'bn', 'cs', 'wg', 'chunks', 'grid_m', 'grid_n', 'xf', 'groups', 'act', 'res', 'out32', 'out16', 'st_tma',
            'phases', 'ctas')
    log = r.stderr.split('SECOND FRAME', 1)[1]
    return [dict(zip(keys, map(int, m.groups()))) for m in LAUNCH_RE.finditer(log)]


def profile_frame(poser, image, poses, options, out_dir):
    """options: {name: value} set for the frame and reset to -1 (automatic) afterwards."""
    from torch.profiler import ProfilerActivity, profile
    ctx = poser.get_context()
    for k, v in options.items():
        ctx.set_option(k, v)
    ctx.set_option('cuda_graphs', 0)          # one kernel record per launch
    with torch.no_grad():
        for i in range(3):
            poser.get_posing_outputs(image, poses[i:i + 1])
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            poser.get_posing_outputs(image, poses[3:4])
            torch.cuda.synchronize()
    ctx.set_option('cuda_graphs', 1)
    for k in options:
        ctx.set_option(k, -1)
    if out_dir:
        tag = '_'.join('%s_%d' % kv for kv in options.items()) or 'auto'
        prof.export_chrome_trace(os.path.join(out_dir, 'halo_layers_%s.pt.trace.json' % tag))
    per = collections.OrderedDict()
    halo = []                                 # (name, us) of every halo launch, in stream order
    for ev in sorted(prof.events(), key=lambda e: e.time_range.start):
        if ev.device_type.name != 'CUDA':
            continue
        t, n = per.get(ev.name, (0.0, 0))
        per[ev.name] = (t + ev.time_range.elapsed_us(), n + 1)
        if halo_split(ev.name):
            halo.append((ev.name, ev.time_range.elapsed_us()))
    profile_frame.halo = halo
    return per


def short(name):
    name = name.replace('(anonymous namespace)::', '').replace('void ', '').replace('tha4::', '')
    return re.sub(r'\(.*$', '', name)


def halo_split(name):
    """conv_halo_kernel<BN, SA, SB, CS, OP, XF, WG, PH, CTAS>: returns (CS, WG) or None."""
    m = re.search(r'conv_halo_kernel<(\d+), (\d+), (\d+), (\d+), (\d+), (\d+), (\d+), (\d+), (\d+)>', name)
    return (int(m.group(4)), int(m.group(7))) if m else None


def print_frame(label, per):
    total = sum(t for t, _ in per.values())
    unsplit = sum(t for k, (t, _) in per.items() if halo_split(k) and halo_split(k)[0] == 1)
    halo = sum(t for k, (t, _) in per.items() if halo_split(k))
    print('\n== one warm teacher_b1 frame, %s: kernel time %.1f us; unsplit halo %.1f us (%.1f %%), all halo %.1f us (%.1f %%)'
          % (label, total, unsplit, 100 * unsplit / total, halo, 100 * halo / total))
    for k, (t, n) in sorted(per.items(), key=lambda kv: -kv[1][0]):
        if t < 0.002 * total:
            continue
        print('  %9.1f us %5.1f %% %4d x  %s' % (t, 100 * t / total, n, short(k)))
    return total, unsplit


def short_launches(shapes, halo, total):
    """The halo launches of the frame with fewer CTAs than SMs: the launch log (shapes, frame order) zipped with the
    halo kernels of the profiled frame (stream order), and their summed device time."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    if len(shapes) != len(halo):
        print('\n== launch log (%d halo launches) and trace (%d) disagree: no per-launch table' % (len(shapes), len(halo)))
        return
    rows = [(s, us) for s, (_, us) in zip(shapes, halo) if s['grid_m'] * s['grid_n'] * s['cs'] < sms]
    print('\n== halo launches of the warm frame with fewer CTAs than SMs (%d), automatic choice' % sms)
    print('  %-28s %3s %3s %3s %6s %5s | %9s' % ('N HxW cin->cout', 'ph', 'wg', 'cs', 'CTAs', 'chnk', 'us'))
    for s, us in rows:
        print('  %-28s %3d %3d %3d %6d %5d | %9.2f' % ('%d %dx%d %d->%d xf%d' % (s['N'], s['H'], s['W'], s['cin'], s['cout'], s['xf']),
              s['phases'], s['wg'], s['cs'], s['grid_m'] * s['grid_n'] * s['cs'], s['chunks'], us))
    short_us = sum(us for _, us in rows)
    print('  %d launches, %.1f us of %.1f us frame kernel time (%.1f %%); of them with 256-pixel or four-phase tiles and '
          '>= 2 chunks: %d launches, %.1f us' % (len(rows), short_us, total, 100 * short_us / total,
                                                sum(1 for s, _ in rows if s['wg'] == 2 and s['chunks'] >= 2),
                                                sum(us for s, us in rows if s['wg'] == 2 and s['chunks'] >= 2)), flush=True)


def shape_ab(shapes, reps):
    import test_gpu_halo_m256 as H
    c = __import__('gpu_util').ctx()
    seen, rows = set(), []
    one_tile = lambda t: t['phases'] == 1 and (t['cs'] == 1 or t['wg'] == 2)       # unsplit, or a row-owning pair
    for s in shapes:
        if not one_tile(s):
            continue
        key = (s['N'], s['H'], s['W'], s['cin'], s['cout'], s['xf'], s['groups'], s['act'], s['res'])
        if key in seen:
            continue
        seen.add(key)
        count = sum(1 for t in shapes if one_tile(t) and (t['N'], t['H'], t['W'], t['cin'], t['cout'], t['xf'], t['groups'], t['act'], t['res']) == key)
        norm = None if not s['xf'] else ('gn' if s['groups'] else 'in')
        inp = H.make_inputs(7, s['N'], s['cin'], s['H'], s['W'], s['cout'], norm, 1 if s['res'] == 1 else 0)
        inp['act'] = s['act'] if s['xf'] else 0
        us = {}
        outs = {}
        try:
            # 128-pixel tiles; 256-pixel, 1 / 2 CTAs per SM; 256-pixel on a row-owning cluster pair (halo_cs = 2)
            for m, (m256, ctas, cs) in enumerate(((0, -1, 1), (1, 1, 1), (1, 2, 1), (1, 1, 2))):
                c.set_option('halo_m256', m256)
                c.set_option('halo_ctas', ctas)
                c.set_option('halo_cs', cs)
                H.conv_norm_ex(**inp, reps=20)                        # warm-up
                y, y16, st, us[m] = H.conv_norm_ex(**inp, reps=reps)
                outs[m] = (y, y16)
        except Exception as e:          # a shape the test hook cannot describe (e.g. Cin not a multiple of 8)
            print('  skipped %s: %s' % (key, e), flush=True)
            continue
        finally:
            c.set_option('halo_m256', -1)
            c.set_option('halo_ctas', -1)
            c.set_option('halo_cs', -1)
        same = all(torch.equal(outs[0][i], outs[m][i]) for m in (1, 2) for i in (0, 1))
        flop = 2.0 * s['N'] * s['H'] * s['W'] * s['cin'] * s['cout'] * 9
        px = s['N'] * s['H'] * s['W']
        hbm = px * s['cin'] * 2 + 9 * s['cin'] * s['cout'] * 2 + px * s['cout'] * (4 + 2) + (px * s['cout'] * 4 if s['res'] == 1 else 0)
        rows.append((s, count, us, flop, hbm, same))
    print('\n== unsplit halo shapes of the frame, alone: %d launches each after warm-up (CUDA events)' % reps)
    print('  %-26s %3s %2s %4s %6s | %9s %7s | %9s %7s %6s | %9s %7s %6s | %9s %7s | %6s %6s %s' % (
        'N HxW cin->cout', 'n', 'cs', 'bn', 'tiles', 'M128 us', 'TFLOP/s', 'M256x1 us', 'TFLOP/s', 'GB/s', 'M256x2 us', 'TFLOP/s', 'GB/s',
        'pair us', 'TFLOP/s', 'x1/x2', 'x1/pr', 'bit-identical'))
    for s, count, us, flop, hbm, same in rows:
        tiles = s['grid_m'] * s['grid_n'] * (2 if s['wg'] == 2 else 1)
        print('  %-26s %3d %2d %4d %6d | %9.2f %7.1f | %9.2f %7.1f %6.0f | %9.2f %7.1f %6.0f | %9.2f %7.1f | %6.3f %6.3f %s' % (
            '%d %dx%d %d->%d xf%d' % (s['N'], s['H'], s['W'], s['cin'], s['cout'], s['xf']), count, s['cs'], s['bn'], tiles,
            us[0], flop / us[0] / 1e6, us[1], flop / us[1] / 1e6, hbm / us[1] / 1e3, us[2], flop / us[2] / 1e6, hbm / us[2] / 1e3,
            us[3], flop / us[3] / 1e6, us[1] / us[2], us[1] / us[3], same))
    return rows


def phase_ab(reps):
    import test_gpu_halo_phase as P
    c = __import__('gpu_util').ctx()
    shapes = [s for s in P.CASES if s[1] == 32 or P.CASES.index(s) < 11]
    # (label, halo_conv, ksplit, halo_ctas, halo_cs)
    paths = (('conv_tc', 0, 0, -1, -1), ('halo x1', 1, 1, 1, 1), ('halo x2', 1, 1, 2, 1), ('pair', 1, 1, 1, 2), ('auto', 1, 0, -1, -1))
    print('\n== four-phase shapes, alone: %d launches each after warm-up (CUDA events); executed TFLOP/s' % reps)
    print('  %-4s %-24s | %s' % ('kind', 'N HxW cin->cout norm', ' | '.join('%10s %7s' % (p[0] + ' us', 'TFLOP/s') for p in paths)) + ' | x1/x2  x1/pr')
    rows = []
    for s in shapes:
        kind, N, Cin, H, W, Cout, norm = s
        inp = P.make_inputs(7, kind, N, Cin, H, W, Cout, norm)
        flop = 2.0 * N * H * W * 16 * Cin * Cout
        us = {}
        try:
            for label, halo, ksplit, ctas, cs in paths:
                c.set_option('halo_conv', halo)
                c.set_option('halo_ctas', ctas)
                c.set_option('halo_cs', cs)
                P.conv_phase(**inp, ksplit=ksplit, reps=20)                  # warm-up
                us[label] = P.conv_phase(**inp, ksplit=ksplit, reps=reps)[3]
        finally:
            c.set_option('halo_conv', 1)
            c.set_option('halo_ctas', -1)
            c.set_option('halo_cs', -1)
        rows.append((s, us))
        print('  %-4d %-24s | %s | %6.3f' % (kind, '%d %dx%d %d->%d %s' % (N, H, W, Cin, Cout, norm), ' | '.join(
            '%10.2f %7.1f' % (us[p[0]], flop / us[p[0]] / 1e6) for p in paths), us['halo x1'] / us['halo x2']) + ' %6.3f' % (us['halo x1'] / us['pair']), flush=True)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=200)
    ap.add_argument('--out', default=None, help='directory for the profiler traces')
    ap.add_argument('--phase-only', action='store_true', help='only the four-phase A/B (step 4)')
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'halo_layers.py needs a CUDA device'
    if args.out:
        os.makedirs(args.out, exist_ok=True)
    print('card:', card(), flush=True)
    if args.phase_only:
        phase_ab(args.reps)
        return
    shapes = frame_shapes()
    print('halo launches in the frame: %d (%d unsplit)' % (len(shapes), sum(1 for s in shapes if s['cs'] == 1)), flush=True)
    poser, image, poses = make_teacher()
    m128 = print_frame('128-pixel tiles (halo_m256 = 0)', profile_frame(poser, image, poses, {'halo_m256': 0}, args.out))
    one = print_frame('one CTA per SM (halo_ctas = 1)', profile_frame(poser, image, poses, {'halo_ctas': 1}, args.out))
    unsplit = print_frame('no cluster pairs (halo_cs = 1)', profile_frame(poser, image, poses, {'halo_cs': 1}, args.out))
    auto = print_frame('automatic choice', profile_frame(poser, image, poses, {}, args.out))
    short_launches(shapes, profile_frame.halo, auto[0])
    print('kernel time per frame: 128-pixel tiles %.1f us, one CTA per SM %.1f us, no cluster pairs %.1f us, automatic %.1f us '
          '(%.3fx over one CTA per SM, %.3fx over no cluster pairs)' % (m128[0], one[0], unsplit[0], auto[0], one[0] / auto[0], unsplit[0] / auto[0]), flush=True)
    shape_ab(shapes, args.reps)
    phase_ab(args.reps)


if __name__ == '__main__':
    main()
