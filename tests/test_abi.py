"""CPU-side checks of the drop-in boundary: the C-ABI library loads and exports every symbol that
include/hvn.h declares; host-side mirrors keep the reference's names and error behaviour."""
import ctypes
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def built_lib():
    from hover_net_b200 import build
    return build.build()


def _declared_symbols():
    src = open(os.path.join(ROOT, "include", "hvn.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(hvn_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol(built_lib):
    L = ctypes.CDLL(built_lib)
    names = _declared_symbols()
    assert len(names) >= 25
    for n in names:
        assert hasattr(L, n), "libhvn.so does not export %s" % n
    assert L.hvn_abi_version() == 1


def test_no_gpu_fails_loudly(built_lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from hover_net_b200 import _lib
    with pytest.raises(_lib.HvnError):
        _lib.Context(0)


def test_product_never_imports_oracle():
    bad = []
    for d, _, files in os.walk(os.path.join(ROOT, "hover_net_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp")):
                txt = open(os.path.join(d, f)).read()
                if re.search(r"^\s*(from|import)\s+oracle\b|libhvo|oracle/|libhvn_probe|conv_probe", txt, flags=re.M):
                    bad.append(f)
    assert not bad, bad


def test_host_spec_matches_reference_key_inventory():
    from hover_net_b200 import arch
    spec = arch.state_dict_spec("original", 5)
    assert list(spec)[0] == "conv0./.weight" and list(spec)[-1] == "upsample2x.unpool_mat"
    n_tracked = sum(k.endswith("num_batches_tracked") for k in spec)
    # variables_tf2pytorch.csv lists 667 keys for the typed model; torch adds num_batches_tracked + unpool_mat
    assert len(spec) - n_tracked - 1 == 667
