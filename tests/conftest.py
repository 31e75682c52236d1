import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, 'tests')):
    if _p not in sys.path:
        sys.path.insert(0, _p)


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs an H100 (run with -m gpu)')


@pytest.fixture(scope='session')
def golden_dir():
    return os.path.join(ROOT, 'tests', 'golden')


@pytest.fixture(scope='session')
def teacher_sds():
    from oracle import synth
    return synth.teacher_state_dicts(0)


@pytest.fixture(scope='session')
def student_sds():
    from oracle import synth
    return synth.student_state_dicts(0)


@pytest.fixture(scope='session')
def lambda00_sds(golden_dir):
    import torch
    return {k: torch.load(os.path.join(golden_dir, 'data', 'lambda_00_%s.pt' % k), map_location='cpu')
            for k in ('face_morpher', 'body_morpher')}


@pytest.fixture(scope='session')
def oracle_clib():
    """The C restatement of the index math (oracle/gridsample_ref.c), built on demand with gcc."""
    import ctypes
    import subprocess
    src = os.path.join(ROOT, 'oracle', 'gridsample_ref.c')
    out_dir = os.path.join(ROOT, 'oracle', '_build')
    out = os.path.join(out_dir, 'libtha4_oracle.so')
    if not os.path.exists(out) or os.path.getmtime(out) < os.path.getmtime(src):
        os.makedirs(out_dir, exist_ok=True)
        subprocess.check_call(['gcc', '-O2', '-ffp-contract=off', '-shared', '-fPIC', '-o', out, src, '-lm'])
    return ctypes.CDLL(out)
