import os
import sys

import numpy as np
import pytest
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if REPO not in sys.path:
    sys.path.insert(0, REPO)
GOLDEN = os.path.join(REPO, 'tests', 'golden')


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (an H100: -m gpu)')


def pytest_collection_modifyitems(config, items):
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason='no CUDA device')
    for item in items:
        if 'gpu' in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope='session')
def golden():
    def load(name):
        return dict(np.load(os.path.join(GOLDEN, name + '.npz'), allow_pickle=False))
    return load


@pytest.fixture(scope='session')
def asset_dir(tmp_path_factory):
    from dynaboa_b200 import config, synthetic
    root = str(tmp_path_factory.mktemp('dboa_assets'))
    synthetic.write_asset_dir(root)
    config.set_data_root(root)
    return root


def rel_err(a, b):
    a = torch.as_tensor(a).double().cpu()
    b = torch.as_tensor(b).double().cpu()
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-30)).item()
