"""CPU-side checks of the drop-in boundary: the C-ABI library loads, exports every symbol
include/nlam_b200.h declares, and the host-side mirror refuses CPU tensors loudly."""
import ctypes
import os
import re

import pytest
import torch

import neural_lam_b200 as nlb
from neural_lam_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    text = open(os.path.join(ROOT, "include", "nlam_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(nlam_[a-z0-9_]+)\s*\(", text)))


def test_library_loads_at_abi_version_3_and_exports_every_declared_symbol():
    L = ctypes.CDLL(_lib.LIB_PATH)
    names = _declared_symbols()
    assert len(names) >= 20
    for n in names:
        assert hasattr(L, n), f"{n} declared in include/nlam_b200.h but not exported"
        assert n in _lib.SYMBOLS, f"{n} has no ctypes prototype"
    assert set(_lib.SYMBOLS) == set(names)
    assert _lib.lib().nlam_abi_version() == 3
    assert b"sm_90a" in _lib.lib().nlam_build_info()


def test_struct_layout_matches_header():
    # NlamMlp: 2 int32 + 4 int32 + 4 ptr + 4 ptr + 2 ptr + float + pad = 24 + 80 + 8 = 112
    assert ctypes.sizeof(_lib.NlamMlp) == 112
    assert ctypes.sizeof(_lib.NlamRowSrc) == 32


def test_cpu_tensors_raise_no_fallback():
    ei = torch.tensor([[0, 1, 2, 0], [1, 0, 1, 2]])
    net = nlb.InteractionNet(ei, 8)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        net(torch.randn(3, 8), torch.randn(3, 8), torch.randn(4, 8))
    mlp = nlb.make_mlp([4, 8, 8])
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        mlp(torch.randn(5, 4))


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_graph_create_without_gpu_fails_loudly():
    ei = torch.tensor([[0, 1, 2, 0], [1, 0, 1, 2]])
    h = ctypes.c_void_p()
    rc = _lib.lib().nlam_graph_create(ctypes.byref(h), ei.contiguous().data_ptr(), 4, 0, 0)
    assert rc == 3  # NLAM_E_CUDA
    assert b"cuda" in _lib.lib().nlam_last_error().lower()
