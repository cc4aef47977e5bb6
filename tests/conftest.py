import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (an H100: run with -m gpu)')


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason='no CUDA device')
    for item in items:
        if 'gpu' in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope='session')
def network_g():
    import yaml
    with open(os.path.join(ROOT, 'options', 'release_test_stage_IIII_dont_need_align_version.yml')) as f:
        return yaml.safe_load(f)['network_g']


@pytest.fixture(scope='session')
def arch_spec(network_g):
    from pgtformer_b200.spec import build_spec
    return build_spec(network_g)


@pytest.fixture(scope='session')
def synth_sd(arch_spec):
    from pgtformer_b200.weights import synth_state_dict
    return synth_state_dict(arch_spec[1], 0)


def load_golden(name):
    import torch
    return torch.load(os.path.join(ROOT, 'tests', 'golden', name), map_location='cpu')


def golden_sample(t, g, key):
    """The elements of t that golden record g keeps for `key` (oracle/make_golden.py: a strided flat sample of the
    reference tensor, whose full shape t must have)."""
    assert tuple(t.shape) == tuple(g[key + '_shape']), (tuple(t.shape), g[key + '_shape'])
    return t.float().cpu().reshape(-1)[::g[key + '_stride']]
