"""The C-ABI library loads on a CPU-only host and exports every symbol include/stmp.h declares; argument
validation that needs no GPU is exercised (no compute calls)."""
import ctypes
import os
import re

import pytest

from pytorch_geometric_temporal_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, "include", "stmp.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(stmp_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    h = ctypes.CDLL(_lib.LIB_PATH)
    names = _declared()
    assert len(names) >= 18
    for n in names:
        assert hasattr(h, n), f"{n} declared in include/stmp.h but not exported"
    assert sorted(_lib.exported_symbols()) == names  # the ctypes table covers exactly the header


def test_version_and_error_channel():
    l = _lib.lib()
    assert l.stmp_version().decode().startswith("stmp ") and "sm_90a" in l.stmp_version().decode()
    # NULL plan -> EINVAL with a message, no CUDA call needed
    rc = l.stmp_spmm(None, 0, 0, 1, 1, None, 1, 1, None, 1, 1, 1.0, None, 0, 0, 0.0, None, None)
    assert rc == _lib.STMP_EINVAL and "plan is NULL" in _lib.last_error()
    with pytest.raises(ValueError):
        _lib.check(rc)
    out = ctypes.c_void_p()
    rc = l.stmp_plan_create(99, 10, 0, None, None, 0, -1.0, 0, None, ctypes.byref(out))
    assert rc == _lib.STMP_EINVAL and "flavor" in _lib.last_error()
    rc = l.stmp_plan_create(_lib.FLAVOR_CHEB, 10, 0, None, None, 7, -1.0, 0, None, ctypes.byref(out))
    assert rc == _lib.STMP_EINVAL and "normalization" in _lib.last_error()
    assert l.stmp_dcrnn_seq_supported(None, 2, 32, 2) == 0
    assert l.stmp_launch_count() >= 0


def test_modules_refuse_cpu_tensors():
    import torch
    from pytorch_geometric_temporal_b200.nn.recurrent import DCRNN
    m = DCRNN(2, 8, 2)
    with pytest.raises(RuntimeError, match="CUDA only"):
        m(torch.randn(4, 2), torch.tensor([[0, 1], [1, 0]]))


def test_state_dict_layout_matches_reference():
    from pytorch_geometric_temporal_b200.nn.recurrent import DCRNN, BatchedDCRNN
    for cls in (DCRNN, BatchedDCRNN):
        sd = cls(2, 32, 3).state_dict()
        assert list(sd) == ["conv_x_z.weight", "conv_x_z.bias", "conv_x_r.weight", "conv_x_r.bias",
                            "conv_x_h.weight", "conv_x_h.bias"]
        assert sd["conv_x_z.weight"].shape == (2, 3, 34, 32) and sd["conv_x_h.bias"].shape == (32,)
    with pytest.raises(AssertionError):
        DCRNN(2, 8, 0)  # assert K > 0 (dcrnn.py:23)
