"""pytest configuration: registers the ``gpu`` marker and shared helpers."""
import glob
import json
import os
import sys

import numpy as np
import pytest
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if REPO not in sys.path:
    sys.path.insert(0, REPO)

GOLDEN_DIR = os.path.join(REPO, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device")


def pytest_collection_modifyitems(config, items):
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


def load_golden(path):
    """-> (meta, state_dict, input, outputs, taps) as torch tensors."""
    z = np.load(path)
    meta = json.loads(bytes(z["meta"]).decode())
    sd, outs, taps = {}, {}, {}
    for k in z.files:
        if k.startswith("sd/"):
            sd[k[3:]] = torch.from_numpy(z[k])
        elif k.startswith("out/"):
            outs[k[4:]] = torch.from_numpy(z[k])
        elif k.startswith("tap/"):
            taps[k[4:]] = torch.from_numpy(z[k])
    return meta, sd, torch.from_numpy(z["input"]), outs, taps


def golden_cases():
    return sorted(glob.glob(os.path.join(GOLDEN_DIR, "case_*.npz")))


@pytest.fixture(params=golden_cases(), ids=lambda p: os.path.basename(p)[5:-4])
def golden(request):
    return load_golden(request.param)
