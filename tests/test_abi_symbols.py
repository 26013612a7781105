"""CPU: the C-ABI library builds for sm_90a, loads, and exports exactly the symbols
declared in include/chgnet_b200.h (no compute calls without a GPU)."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as entry

    entry.build()
    from chgnet_b200 import _lib

    return _lib.load_library()


def _declared():
    src = open(os.path.join(ROOT, "include", "chgnet_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(chg_[a-z0-9_]+)\s*\(", src)))


def test_header_symbols_are_exported(lib):
    names = _declared()
    assert len(names) >= 20
    for name in names:
        assert hasattr(lib, name), f"{name} declared in the header but not exported"


def test_binding_table_matches_header(lib):
    from chgnet_b200 import _lib

    declared = set(_declared()) - {"chg_last_error", "chg_abi_version", "chg_launch_count", "chg_set_option",
                                   "chg_wgrad_workspace_floats", "chg_gated_fused_workspace_floats", "chg_packed_floats", "chg_pack_weights_host",
                                   "chg_forward_plan", "chg_forward",
                                   "chg_graph_build", "chg_graph_sizes", "chg_graph_export", "chg_graph_free",
                                   "chg_graph_build_many", "chg_graph_views", "chg_graph_free_many",
                                   "chg_pack_batch_host", "chg_pack_batch_wire", "chg_host_alloc", "chg_host_free", "chg_build_csr", "chg_build_csr_scratch_ints", "chg_bond_graph_count",
                                   "chg_graph_build_device", "chg_graph_device_scratch_bytes", "chg_md_kick_drift", "chg_md_kick",
                                   "chg_fire_step"}
    assert declared == set(_lib.SIGNATURES)
    # argument counts of the ctypes table follow the header prototypes
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "chgnet_b200.h")).read(), flags=re.S)
    for name, argtypes in _lib.SIGNATURES.items():
        proto = re.search(rf"int {name}\s*\((.*?)\);", src, flags=re.S).group(1)
        assert len(proto.split(",")) == len(argtypes), name


def test_scratch_chunk_counts_match_header():
    """The wrappers size the kernels' scratch from copies of the header's chunk limits: a copy smaller than its
    #define would let the kernels write past the scratch."""
    from chgnet_b200 import _lib

    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "chgnet_b200.h")).read(), flags=re.S)
    for name in ("DOS_MAX_CHUNKS", "TD_MAX_CHUNKS", "JDOS_MAX_CHUNKS"):
        value = int(re.search(rf"#define CHG_{name}\s+(\d+)", src).group(1))
        assert getattr(_lib, name) == value, name


def test_library_metadata(lib):
    assert lib.chg_abi_version() == 3
    assert lib.chg_launch_count() >= 0
    assert lib.chg_last_error() is not None


def test_product_fails_loudly_without_cuda():
    import torch

    if torch.cuda.is_available():
        pytest.skip("CUDA present")
    from chgnet_b200._lib import ChgnetB200Error, CudaKernels
    from chgnet_b200.model import CHGNet

    with pytest.raises(ChgnetB200Error, match="CUDA device"):
        CudaKernels()
    model = CHGNet.from_file(os.path.join(ROOT, "tests", "golden", "chgnet_0.3.0_weights.npz"))
    with pytest.raises(RuntimeError, match="no CPU path"):
        model([])


def test_sass_is_sm90a():
    so = os.path.join(ROOT, "chgnet_b200", "libchgnet_b200.so")
    import subprocess

    out = subprocess.run(["cuobjdump", "-lelf", so], capture_output=True, text=True).stdout
    assert "sm_90a" in out, out


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, "chgnet_b200")
    for fn in os.listdir(pkg):
        if fn.endswith(".py"):
            assert "oracle" not in open(os.path.join(pkg, fn)).read().replace("the oracle", "").replace("oracle.kernel_specs.SpecKernels", ""), fn
