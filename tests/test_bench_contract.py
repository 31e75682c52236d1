"""bench.py contract checks that need no GPU: the reference arm runs here (CPU port of the reference path) and prints
exactly one JSON line with the agreed keys; --dump-outputs writes float32 arrays within its size budget."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BASE_KEYS = {'metric', 'value', 'unit', 'n_gpus', 'steps', 'warmup', 'ms_per_step', 'higher_is_better', 'scaling', 'vs_baseline',
             'dtype', 'data', 'config'}


def test_reference_arm_prints_one_json_line():
    env = dict(os.environ, THA4_CPU_THREADS='8')
    out = subprocess.run([sys.executable, os.path.join(ROOT, 'bench.py'), '--impl', 'reference', '--steps', '1', '--warmup', '3'],
                         capture_output=True, text=True, timeout=600, env=env, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    lines = [l for l in out.stdout.splitlines() if l.strip()]
    assert len(lines) == 1, lines
    d = json.loads(lines[0])
    assert d['impl'] == 'reference' and BASE_KEYS <= set(d)
    assert d['metric'] == '512x512 RGBA frames/sec' and d['unit'] == 'frames/s' and d['higher_is_better'] is True
    assert d['value'] > 0 and d['cpu_baseline']['kind'] in ('port', 'reference') and d['cpu_baseline']['cores'] >= 1
    assert d['e2e'] == {'value': d['value'], 'unit': 'frames/s', 'h2d_bytes_per_step': 0, 'd2h_bytes_per_step': 0}


def test_dump_outputs_writes_float32_within_budget(tmp_path):
    sys.path.insert(0, ROOT)
    import numpy as np
    import torch
    import bench
    big = {'a': torch.arange(3 * 1024 * 1024 * 4, dtype=torch.float32).reshape(4, -1), 'b': torch.ones(2, 3, dtype=torch.float64)}
    limit = bench.DUMP_LIMIT_BYTES
    bench.DUMP_LIMIT_BYTES = 1 << 20
    try:
        bench.dump_outputs(str(tmp_path / 'x'), big)
        bench.dump_outputs(str(tmp_path / 'y'), big)
    finally:
        bench.DUMP_LIMIT_BYTES = limit
    a, b = np.load(tmp_path / 'x' / 'a.npy'), np.load(tmp_path / 'x' / 'b.npy')
    assert a.dtype == np.float32 and b.dtype == np.float32 and a.nbytes + b.nbytes <= 1 << 20
    assert np.array_equal(a, np.load(tmp_path / 'y' / 'a.npy'))           # the same seeded sample every run
    assert np.all(np.diff(a) > 0) and b.shape == (2, 3)                    # sorted indices of arange; small tensors stay whole
