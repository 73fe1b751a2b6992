"""CPU side of ASTGCN on 321 .. 1024 nodes: the PeMS03 / PeMS07-shaped generators, the golden fixture of
tests/golden/make_goldens_astgcn_large.py (self-consistent, reproducible from its seeds) and the float64 oracle against it."""
import gzip
import os

import numpy as np
import pytest
import torch

from oracle import attention as A
from pytorch_geometric_temporal_b200.dataset import synthetic
from pytorch_geometric_temporal_b200.nn.attention import ASTGCN

GRAPHS = {"pems07": (synthetic.pems07_like, 883, 866), "pems03": (synthetic.pems03_like, 358, 547)}


@pytest.fixture(scope="module")
def golden(golden_dir):
    with gzip.open(os.path.join(golden_dir, "astgcn_large.pt.gz"), "rb") as f:
        return torch.load(f, weights_only=False)


@pytest.mark.parametrize("graph", sorted(GRAPHS))
def test_pems_like_generators(graph):
    like, n, links = GRAPHS[graph]
    e = like(0)
    assert e.dtype == np.int64 and e.shape == (2, 2 * links)
    assert e.min() >= 0 and e.max() < n
    assert np.all(e[0] != e[1])                                             # no self loops
    keys = e[0] * n + e[1]
    assert len(np.unique(keys)) == e.shape[1]                               # no duplicates
    assert np.array_equal(np.sort(keys), np.sort(e[1] * n + e[0]))          # symmetric
    assert np.all(np.diff(keys) > 0)                                        # row-major order
    assert np.array_equal(e, like(0)) and not np.array_equal(e, like(1))    # seeded


def test_golden_fixture_is_self_consistent(golden):
    assert set(golden["cases"]) == {"pems07_sym", "pems07_none", "pems03_sym"}
    for name, c in golden["cases"].items():
        like, n, links = GRAPHS[c["graph"]]
        assert torch.equal(c["edge_index"], torch.from_numpy(like(c["graph_seed"])))
        B = c["X"].size(0)
        assert c["X"].shape == (B, n, 1, 12) and c["out"].shape == (B, n, 12)
        assert torch.equal(c["X"], torch.randn(B, n, 1, 12, generator=torch.Generator().manual_seed(c["x_seed"])))
        assert torch.isfinite(c["out"]).all()
        torch.manual_seed(c["seed"])
        m = ASTGCN(**golden["ctor"], num_of_vertices=n, normalization=c["normalization"])
        chk = float(sum(v.double().abs().sum() for v in m.state_dict().values()))
        assert abs(chk - c["state_checksum"]) <= 1e-6 * c["state_checksum"], name


@pytest.mark.parametrize("case", ["pems03_sym", "pems07_none"])
def test_oracle_matches_golden(golden, case):
    """the functional restatement (oracle/attention.py) in float64 reproduces the reference's float64 output"""
    c = golden["cases"][case]
    n = c["X"].size(1)
    torch.manual_seed(c["seed"])
    m = ASTGCN(**golden["ctor"], num_of_vertices=n, normalization=c["normalization"])
    p = {k: v.double() for k, v in m.state_dict().items()}
    X = c["X"][:2].double()
    with torch.no_grad():
        got = A.astgcn(p, X, c["edge_index"], 3, c["normalization"], 1)
    want = c["out"][:2].double()
    assert got.shape == want.shape
    assert torch.allclose(got, want, rtol=1e-5, atol=1e-6), (got - want).abs().max().item()
