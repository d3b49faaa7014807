import json
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]
GOLDEN = ROOT / "tests" / "golden"
for p in (str(ROOT), str(ROOT / "k-diffusion_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def pytest_collection_modifyitems(config, items):
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


def unhex(h):
    """list of 8-hex-digit fp32 bit patterns -> fp32 tensor"""
    return torch.tensor([int(v, 16) for v in h], dtype=torch.int64).to(torch.int32).view(torch.float32) if h else torch.zeros(0)


def bits(t):
    return [format(int(v) & 0xFFFFFFFF, "08x") for v in t.detach().float().cpu().contiguous().view(torch.int32).flatten().tolist()]


@pytest.fixture(scope="session")
def kat():
    return json.loads((GOLDEN / "kat.json").read_text())


def load_npz(name):
    with np.load(GOLDEN / name) as z:
        return {k: torch.from_numpy(z[k]) for k in z.files}


def load_fixture(stem):
    """(config dict after reference load_config defaults, {key: shape}, tensors)"""
    meta = json.loads((GOLDEN / f"{stem}_shapes.json").read_text())
    return meta["config"], meta["shapes"], load_npz(f"{stem}.npz")


from oracle.fixtures import assert_close, synth_sd  # noqa: E402,F401
