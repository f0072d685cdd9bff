"""The C-ABI boundary without a GPU: the library builds for sm_90a, loads, and exports exactly the symbols include/focoos_b200.h declares;
the Python marshalling layer binds all of them; host-only entry points work; compute entry points refuse CPU tensors (no fallback)."""
import ctypes
import os
import re
import subprocess

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "focoos_b200.h")
LIB = os.path.join(ROOT, "focoos_b200", "lib", "libfocoos_b200.so")


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as g

    g.build()  # cached by a source hash; cross-compiles with nvcc when something changed
    return ctypes.CDLL(LIB)


def declared_symbols():
    text = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    return sorted(set(re.findall(r"\b(fb200_[a-z0-9_]+)\s*\(", text)))


def test_header_symbols_are_exported(lib):
    names = declared_symbols()
    assert len(names) >= 60
    for n in names:
        assert hasattr(lib, n), f"{n} is declared in include/focoos_b200.h but not exported by {LIB}"
    nm = subprocess.run(["nm", "-D", "--defined-only", LIB], capture_output=True, text=True, check=True).stdout
    exported = sorted(set(re.findall(r" T (fb200_[a-z0-9_]+)", nm)))
    assert exported == names, (sorted(set(exported) - set(names)), sorted(set(names) - set(exported)))


def test_python_layer_binds_every_symbol(lib):
    from focoos_b200 import autograd_ops, criterion, ops, train_step  # noqa: F401  (each module appends its entry points)

    assert sorted(ops.EXPORTED_SYMBOLS) == declared_symbols()


def test_host_only_entry_points(lib):
    lib.fb200_last_error.restype = ctypes.c_char_p
    assert lib.fb200_version() >= 1
    lib.fb200_optim_workspace_bytes.restype = ctypes.c_int64
    lib.fb200_detr_loss_workspace_bytes.restype = ctypes.c_int64
    lib.fb200_col_workspace_bytes.restype = ctypes.c_int64
    assert lib.fb200_optim_workspace_bytes() > 0 and lib.fb200_detr_loss_workspace_bytes(7, 16, 300) > 0 and lib.fb200_col_workspace_bytes(256) > 0
    assert lib.fb200_conv_wgrad_tc_supported(16, 80, 80, 256, 80, 80, 256, 3, 3, 1, 1) == 1
    assert lib.fb200_conv_wgrad_tc_supported(16, 80, 80, 256, 40, 40, 256, 3, 3, 2, 1) == 1
    assert lib.fb200_conv_wgrad_tc_supported(16, 640, 640, 3, 320, 320, 32, 3, 3, 2, 1) == 0  # 3 channels: CUDA-core kernel
    # argument validation happens before any CUDA call: a null pointer is an error with a message, not a crash
    rc = lib.fb200_topk(None, 1, 10, 3, None, None, None)
    assert rc < 0 and b"topk" in lib.fb200_last_error()


def test_ops_refuse_cpu_tensors():
    from focoos_b200 import ops

    x = torch.zeros((1, 4, 4, 32))
    with pytest.raises(RuntimeError):
        ops.conv2d(x, torch.zeros((32, 1, 1, 32)))
    with pytest.raises(RuntimeError):
        ops.maxpool3x3s2(x)
