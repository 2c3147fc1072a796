"""The C-ABI shared library loads and exports every symbol include/dfvo_b200.h declares; no compute
calls (runs without a GPU).  The nvcc-built product library is checked when present (it is built by
__graft_entry__.build()), the host-emulation build always."""
import os
import re

import pytest

from b200 import native

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    txt = open(os.path.join(ROOT, "include", "dfvo_b200.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(dfvo_[a-z0-9_]+)\s*\(", txt)))


def test_header_and_binding_table_agree():
    syms = header_symbols()
    assert len(syms) >= 25
    assert sorted(native.SIGNATURES) == syms


def test_hostsim_library_exports_all(hostsim_lib):
    for s in header_symbols():
        assert hasattr(hostsim_lib.cdll, s)
    assert hostsim_lib.dfvo_is_device_build() == 0


def test_product_library_exports_all_and_is_device_build():
    if not os.path.exists(native.LIB_PATH):
        pytest.skip("libdfvo_b200.so not built yet (run __graft_entry__.build())")
    lib = native.Lib(native.LIB_PATH)                     # dlopen only: needs libcudart, not a GPU
    for s in header_symbols():
        assert hasattr(lib.cdll, s)
    assert lib.dfvo_is_device_build() == 1
    assert b"sm_90a" in lib.dfvo_version()


def test_product_loader_refuses_without_cuda():
    import torch
    if torch.cuda.is_available():
        pytest.skip("CUDA present")
    with pytest.raises(native.DfvoError):
        native.require_cuda()
