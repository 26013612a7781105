import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def pytest_collection_modifyitems(config, items):
    """`-m gpu` tests need a CUDA device: on a CPU-only host they are skipped, not failed (a plain
    `pytest tests/` stays green on a machine without a GPU)."""
    import torch

    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device visible")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def weights030():
    from oracle import chgnet_oracle as orc

    return orc.load_weights_npz(os.path.join(GOLDEN_DIR, "chgnet_0.3.0_weights.npz"))


@pytest.fixture(scope="session")
def golden():
    import numpy as np

    with np.load(os.path.join(GOLDEN_DIR, "chgnet_0.3.0_golden.npz")) as f:
        return {k: f[k] for k in f.files}


@pytest.fixture(scope="session")
def limno2_graph(golden):
    import torch

    from chgnet_b200.graph import CrystalGraph

    g = {k.split("limno2.graph.")[1]: torch.from_numpy(v) for k, v in golden.items() if k.startswith("limno2.graph.")}
    return CrystalGraph(atom_graph_cutoff=6.0, bond_graph_cutoff=3.0, graph_id="mp-18767", **g)
