import glob
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN_DIR = os.path.join(ROOT, 'tests', 'golden')


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (an H100)')


def pytest_collection_modifyitems(config, items):
    """`gpu`-marked tests need a CUDA device: on a machine without one they are skipped, not failed (a bare
    `pytest tests` must be green there too)."""
    try:
        import torch
        has = torch.cuda.is_available()
    except Exception:
        has = False
    if has:
        return
    skip = pytest.mark.skip(reason='no CUDA device on this machine')
    for item in items:
        if 'gpu' in item.keywords:
            item.add_marker(skip)


def golden_names():
    return sorted(os.path.basename(f)[:-4] for f in glob.glob(os.path.join(GOLDEN_DIR, '*.npz')))


def load_golden(name):
    """Returns dict(guidance, blur, sparse_depth|None, prop_time, norm_type, out) as numpy arrays.
    Large cases regenerate their inputs from the recorded seed (cspn_b200.synth, CPU generator)."""
    from cspn_b200.synth import make_inputs
    z = np.load(os.path.join(GOLDEN_DIR, name + '.npz'))
    if 'guidance' in z:
        g, d = z['guidance'], z['blur']
        sp = z['sparse_depth'] if 'sparse_depth' in z else None
    else:
        s = str(z['sparse'])
        g, d, sp = make_inputs(int(z['seed']), int(z['B']), int(z['C']), int(z['H']), int(z['W']), int(z['gch']),
                               None if s == 'None' else s, int(z['n_sample']))
        g, d, sp = g.numpy(), d.numpy(), (None if sp is None else sp.numpy())
    return dict(guidance=g, blur=d, sparse_depth=sp, prop_time=int(z['prop_time']),
                norm_type=str(z['norm_type']), out=z['out'])


@pytest.fixture(scope='session')
def has_cuda():
    import torch
    return torch.cuda.is_available()
