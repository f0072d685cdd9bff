"""The C-ABI boundary without a GPU: the library builds for sm_90a, loads, and exports exactly the symbols include/focoos_b200.h declares;
the Python marshalling layer types all of them from the header and calls each with its declared arity; the CPU reference backend mirrors the
CUDA backend's methods; host-only entry points work; compute entry points refuse CPU tensors (no fallback)."""
import ast
import ctypes
import inspect
import os
import re
import subprocess

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "focoos_b200.h")
LIB = os.path.join(ROOT, "focoos_b200", "lib", "libfocoos_b200.so")
OPS = os.path.join(ROOT, "focoos_b200", "ops.py")


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as g

    g.build()  # cached by a source hash; cross-compiles with nvcc when something changed
    return ctypes.CDLL(LIB)


def declared_symbols():
    text = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    return sorted(set(re.findall(r"\b(fb200_[a-z0-9_]+)\s*\(", text)))


def declared_param_counts():
    """{name: number of parameters} of every declaration, read from the header independently of ops.parse_header"""
    text = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    return {n: 0 if a.strip() in ("", "void") else a.count(",") + 1 for n, a in re.findall(r"\b(fb200_[a-z0-9_]+)\s*\(([^)]*)\)", text)}


def test_header_symbols_are_exported(lib):
    names = declared_symbols()
    assert len(names) >= 60
    for n in names:
        assert hasattr(lib, n), f"{n} is declared in include/focoos_b200.h but not exported by {LIB}"
    nm = subprocess.run(["nm", "-D", "--defined-only", LIB], capture_output=True, text=True, check=True).stdout
    exported = sorted(set(re.findall(r" T (fb200_[a-z0-9_]+)", nm)))
    assert exported == names, (sorted(set(exported) - set(names)), sorted(set(names) - set(exported)))


def test_load_library_types_every_declared_symbol(lib):
    from focoos_b200 import ops

    bound = {n: f for n, f in vars(ops.load_library()).items() if n.startswith("fb200_")}
    assert sorted(bound) == declared_symbols()
    counts = declared_param_counts()
    for n, f in bound.items():
        assert f.argtypes is not None and len(f.argtypes) == counts[n], (n, f.argtypes, counts[n])
        if n == "fb200_last_error":
            assert f.restype is ctypes.c_char_p
        elif n.endswith("_workspace_bytes"):
            assert f.restype is ctypes.c_int64, n
        else:
            assert f.restype is ctypes.c_int, n
    # fb200_layernorm(x, res, gamma, beta, out, int dtype, int64_t M, int C, float eps, void* stream)
    assert bound["fb200_layernorm"].argtypes == [ctypes.c_void_p] * 5 + [ctypes.c_int, ctypes.c_int64, ctypes.c_int, ctypes.c_float, ctypes.c_void_p]


def test_backend_calls_match_the_header():
    """every call of an entry point in ops.py - `self._call("fb200_...", ...)` and direct `lib.fb200_...(...)` - names a declared symbol and passes exactly
    its parameter count; every declared symbol is called there"""
    counts = declared_param_counts()
    used, launches = set(), 0
    for node in ast.walk(ast.parse(open(OPS).read())):
        if not isinstance(node, ast.Call) or not isinstance(node.func, ast.Attribute):
            continue
        if node.func.attr == "_call":
            first, args = node.args[0], node.args[1:]
            names = [first.body.value, first.orelse.value] if isinstance(first, ast.IfExp) else [first.value]  # stem_conv picks the uint8 variant
            launches += 1
        elif node.func.attr.startswith("fb200_"):
            names, args = [node.func.attr], node.args
        else:
            continue
        assert not node.keywords and not any(isinstance(a, ast.Starred) for a in args), ast.unparse(node)
        for n in names:
            assert n in counts, f"{n} is not declared in include/focoos_b200.h"
            assert len(args) == counts[n], f"{n}: {len(args)} arguments, the header declares {counts[n]}"
            used.add(n)
    assert launches >= 70
    # fb200_version is an integration query with no use on the operator path (test_host_only_entry_points calls it)
    assert set(counts) - used == {"fb200_version"}


def test_header_parser_rejects_unknown_types():
    from focoos_b200 import ops

    assert ops.parse_header("int64_t fb200_x(const float* a, int b, float c, void* s);") == {"fb200_x": (ctypes.c_int64, [ctypes.c_void_p, ctypes.c_int, ctypes.c_float, ctypes.c_void_p])}
    with pytest.raises(ValueError, match="double"):
        ops.parse_header("int fb200_x(double a);")
    with pytest.raises(ValueError, match="double"):
        ops.parse_header("double fb200_x(void);")


def test_reference_backend_mirrors_the_cuda_backend():
    from focoos_b200.ops import CudaBackend
    from oracle.ops_ref import RefBackend

    def public(cls):
        return {n: inspect.signature(getattr(cls, n)) for n in dir(cls) if not n.startswith("_") and callable(getattr(cls, n))}

    cuda, ref = public(CudaBackend), public(RefBackend)
    assert sorted(cuda) == sorted(ref), (sorted(set(cuda) - set(ref)), sorted(set(ref) - set(cuda)))
    assert len(cuda) >= 70
    for n in cuda:
        assert cuda[n] == ref[n], (n, str(cuda[n]), str(ref[n]))


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
