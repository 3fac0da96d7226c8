"""CPU-side checks of the C-ABI boundary: the shared library loads without a GPU and exports every symbol that
include/seg_b200.h declares (no compute calls here)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "seg_b200.h")
LIB = os.path.join(ROOT, "pytorch-segmentation_b200", "libseg_b200.so")


def declared_symbols():
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(seg_[a-z0-9_]+)\s*\(", src)))


@pytest.fixture(scope="module")
def cdll():
    if not os.path.exists(LIB):
        import __graft_entry__
        __graft_entry__.build()
    return ctypes.CDLL(LIB)


def test_header_declares_entry_points():
    syms = declared_symbols()
    assert len(syms) >= 30
    for must in ("seg_conv2d_fwd", "seg_conv2d_dgrad", "seg_conv2d_wgrad", "seg_bn_finalize", "seg_upsample_loss_fwd",
                 "seg_loss_nchw_fwd", "seg_last_error"):
        assert must in syms


def test_library_exports_every_declared_symbol(cdll):
    missing = [s for s in declared_symbols() if not hasattr(cdll, s)]
    assert not missing, f"declared in include/seg_b200.h but not exported: {missing}"


def test_python_binding_matches_header(cdll):
    from seg_b200 import lib
    declared = set(declared_symbols())
    bound = set(lib.EXPORTS)
    assert bound <= declared, f"bound but not declared: {sorted(bound - declared)}"
    lib.load()
    assert lib.load().seg_version() >= 100


def test_conv_desc_layout_matches_header():
    from seg_b200 import lib
    assert ctypes.sizeof(lib.ConvDesc) == 14 * 4
    assert ctypes.sizeof(lib.SyncDesc) == 32  # pointer, three int32, padding, int64: static_assert'ed in csrc/seg_comm.cu
    d = lib.make_conv_desc(2, 33, 33, 2048, 256, 3, 3, 1, 18, 18)
    assert (d.P, d.Q) == (33, 33)
    d = lib.make_conv_desc(1, 513, 513, 3, 64, 7, 7, 2, 3, 1)
    assert (d.P, d.Q) == (257, 257)


def test_product_package_never_imports_the_oracle():
    """oracle/ is test infrastructure: nothing under pytorch-segmentation_b200/ (host package, overlay, kernels) may import,
    include or execute it — the product path has no CPU restatement to fall back to."""
    pkg = os.path.join(ROOT, "pytorch-segmentation_b200")
    offenders = []
    for d, _, files in os.walk(pkg):
        if os.path.basename(d) in ("build", "__pycache__"):
            continue
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".sh")):
                src = open(os.path.join(d, f), errors="ignore").read()
                imports = re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M)          # Python import
                executes = re.search(r"(#include|open\(|exec\(|runpy)[^\n]*oracle/", src)          # include / read / run
                if imports or executes:
                    offenders.append(os.path.relpath(os.path.join(d, f), ROOT))
    assert not offenders, offenders
