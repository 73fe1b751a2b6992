"""Host-side checks of the narrow-state DCRNN: the oracle reproduces the reference goldens it is tested against on the GPU
(tests/golden/make_goldens_narrow.py), and the launch-shape switch is known to the library without a CUDA call."""
import os

import pytest
import torch

from oracle import recurrent as R
from pytorch_geometric_temporal_b200 import _lib


def _load(golden_dir, name):
    return torch.load(os.path.join(golden_dir, name + ".pt"), weights_only=False)


def _params(state):
    return {k: v.clone().requires_grad_(True) for k, v in state.items()}


def _check_grads(p, g):
    for k, v in p.items():
        ref = g["grads"][k]
        assert torch.allclose(v.grad, ref, rtol=1e-4, atol=1e-5 * max(ref.abs().max().item(), 1.0)), k


@pytest.mark.parametrize("name", ["dcrnn_narrow_pems_bay", "dcrnn_narrow_metr_la", "dcrnn_narrow_chickenpox"])
def test_oracle_reproduces_batched_goldens(golden_dir, name):
    g = _load(golden_dir, name)
    p = _params(g["state"])
    X = g["X"].clone().requires_grad_(True)
    out = R.batched_dcrnn(p, X, g["edge_index"], g["edge_weight"])
    assert torch.allclose(out, g["out"], rtol=1e-5, atol=1e-6)
    (out * torch.linspace(-1, 1, out.numel()).view_as(out)).sum().backward()
    assert torch.allclose(X.grad, g["gX"], rtol=1e-4, atol=1e-6)
    _check_grads(p, g)


def test_oracle_reproduces_cell_golden(golden_dir):
    g = _load(golden_dir, "dcrnn_narrow_cell")
    p = _params(g["state"])
    X, H = g["X"].clone().requires_grad_(True), g["H"].clone().requires_grad_(True)
    out = R.dcrnn_cell(p, X, g["edge_index"], g["edge_weight"], H)
    assert torch.allclose(out, g["out"], rtol=1e-5, atol=1e-6)
    (out * torch.linspace(-1, 1, out.numel()).view_as(out)).sum().backward()
    assert torch.allclose(X.grad, g["gX"], rtol=1e-4, atol=1e-6)
    assert torch.allclose(H.grad, g["gH"], rtol=1e-4, atol=1e-6)
    _check_grads(p, g)


def test_narrow_pack_switch_is_host_only():
    for p in (1, 2, 8, 0):
        _lib.set_option("dcrnn_narrow_pack", p)          # no CUDA call behind it
    for bad in (-1, 9):
        with pytest.raises(ValueError):
            _lib.set_option("dcrnn_narrow_pack", bad)
    _lib.set_option("dcrnn_narrow_pack", 0)


def test_narrow_backward_symbols_are_in_the_abi():
    l = _lib.lib()
    assert l.stmp_dcrnn_narrow_bwd_supported(None, 2, 2, 3) == 0
    assert l.stmp_dcrnn_narrow_bwd_seq(None, 1, 1, 2, 2, 3, *([None] * 11)) == _lib.STMP_EINVAL
