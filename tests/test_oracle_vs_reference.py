"""Pin of the oracle's MODULE logic: the functional restatement (oracle/recurrent.py, oracle/attention.py) must reproduce the
UNMODIFIED reference modules bit-for-bit.  The reference modules were run once on these inputs (tests/golden/make_goldens_ref_compare.py):
their state dicts, inputs and outputs are stored in tests/golden/ref_compare.pt.gz."""
import pytest
import torch

from oracle import attention as A, golden, pyg, recurrent as R


def _graph(n=12, e=40, seed=0):
    g = torch.Generator().manual_seed(seed)
    row = torch.randint(0, n, (e,), generator=g)
    col = torch.randint(0, n, (e,), generator=g)
    pairs = {(int(r), int(c)) for r, c in zip(row, col)} | {(i, i) for i in range(n)} | {(i, (i + 1) % n) for i in range(n)}
    ei = torch.tensor(sorted(pairs)).t().contiguous()
    return ei, torch.rand(ei.size(1), generator=g) * 0.9 + 0.1


def _undirected(ei):
    und = sorted({(a, b) for a, b in ei.t().tolist() if a != b} | {(b, a) for a, b in ei.t().tolist() if a != b})
    return torch.tensor(und).t().contiguous()


def _case(key):
    return golden.load()["oracle"][key]


@pytest.mark.parametrize("K", [1, 2, 3, 4])
def test_dcrnn(K):
    ei, ew = _graph()
    c = _case(f"dcrnn_K{K}")
    assert torch.equal(c["out_h"], R.dcrnn_cell(c["sd"], c["X"], ei, ew, c["H"]))
    assert torch.equal(c["out"], R.dcrnn_cell(c["sd"], c["X"], ei))
    assert torch.equal(c["outb"], R.batched_dcrnn(c["sdb"], c["Xb"], ei, ew))


@pytest.mark.parametrize("K", [1, 2, 3, 4])
@pytest.mark.parametrize("norm", ["sym", "rw", None])
def test_gconv(K, norm):
    ei, ew = _graph()
    c = _case(f"gconv_K{K}_{norm}")
    lm = None if norm == "sym" else torch.tensor(2.3)
    X, H, C = c["X"], c["H"], c["C"]
    assert torch.equal(c["gru"], R.gconv_gru_cell(c["sd_gru"], X, ei, ew, H, lm, norm))
    b = R.gconv_lstm_cell(c["sd_lstm"], X, ei, ew, H, C, lm, norm)
    assert torch.equal(c["lstm"][0], b[0]) and torch.equal(c["lstm"][1], b[1])


def test_tgcn_family():
    ei, ew = _graph()
    c = _case("tgcn_family")
    X, H = c["X"], c["H"]
    for improved in (False, True):
        for asl in (True, False):
            sd, want = c[f"tgcn_{improved}_{asl}"]
            assert torch.equal(want, R.tgcn_cell(sd, X, ei, ew, H, improved, asl))
    sd, want = c["tgcn2"]
    assert torch.equal(want, R.tgcn_cell(sd, c["Xb"], ei, ew, c["Hb"]))
    sd, want = c["a3tgcn2"]
    assert torch.equal(want, R.a3tgcn(sd, c["Xp"], ei, ew))
    sd, want = c["a3tgcn"]
    assert torch.equal(want, R.a3tgcn(sd, c["Xp"][0], ei, ew))


@pytest.mark.parametrize("norm", ["sym", None, "rw"])
def test_astgcn(norm):
    ei, _ = _graph()
    eiu = _undirected(ei)
    c = _case(f"astgcn_{norm}")
    lm = None
    if norm != "sym":
        lm = pyg.LaplacianLambdaMax()(pyg.Data(edge_index=eiu, edge_attr=None, num_nodes=12)).lambda_max
        assert torch.equal(torch.as_tensor(lm), torch.as_tensor(c["lm"]))
    got = A.astgcn(c["sd"], c["X"], eiu, 2, norm, 2, lm)
    assert torch.allclose(c["want"], got, rtol=1e-6, atol=1e-6)  # diag-scale vs dense matmul: 1 ulp


@pytest.mark.parametrize("norm", ["sym", None, "rw"])
def test_chebconv_attention_per_graph_lambda_max(norm):
    """The multi-graph mini-batch call of the reference's own test (test/attention_test.py:205-218): a node->graph `batch`
    vector and one lambda_max per graph."""
    c = _case(f"chebatt_{norm}")
    batch = torch.tensor([0, 0, 0, 1, 1, 1, 1])
    ei = torch.tensor([[0, 1, 1, 2, 3, 4, 5, 6, 3, 6], [1, 0, 2, 1, 4, 3, 6, 5, 6, 3]])
    lam = torch.tensor([2.0, 3.0])
    got = A.cheb_conv_attention(c["sd"], c["x"], ei, c["S"], norm, c["ew"], lam, batch)
    assert torch.allclose(c["want"], got, rtol=1e-6, atol=1e-6)
    assert not torch.allclose(c["want"], c["want_one_lambda"], rtol=1e-3, atol=1e-4)   # the second graph really uses 3.0


# ---- SURVEY 8f rank 1: GCLSTM, STConv, MSTGCN ---------------------------------------------------------------
@pytest.mark.parametrize("K", [1, 2, 3])
@pytest.mark.parametrize("norm", ["sym", "rw", None])
def test_gc_lstm(K, norm):
    ei, ew = _graph()
    c = _case(f"gc_lstm_K{K}_{norm}")
    lm = None if norm == "sym" else torch.tensor(2.3)
    b = R.gc_lstm_cell(c["sd"], c["X"], ei, ew, c["H"], c["C"], lm, norm)
    assert torch.equal(c["full"][0], b[0]) and torch.equal(c["full"][1], b[1])
    b = R.gc_lstm_cell(c["sd"], c["X"], ei, lambda_max=lm, normalization=norm)
    assert torch.equal(c["bare"][0], b[0]) and torch.equal(c["bare"][1], b[1])


@pytest.mark.parametrize("K", [1, 2, 3])
def test_stconv(K):
    ei, ew = _graph()
    c = _case(f"stconv_K{K}")
    X = c["X"]
    assert torch.equal(c["train"], A.stconv({k: v.clone() for k, v in c["sd_train"].items()}, X, ei, ew))   # training-mode BatchNorm
    assert torch.equal(c["eval"], A.stconv(c["sd_eval"], X, ei, ew, training=False))
    assert torch.equal(c["tconv1"], A.temporal_conv({k[len("_temporal_conv1."):]: v for k, v in c["sd_eval"].items()
                                                     if k.startswith("_temporal_conv1.")}, X))


@pytest.mark.parametrize("strides", [1, 2])
def test_mstgcn(strides):
    ei, _ = _graph()
    eiu = _undirected(ei)
    c = _case(f"mstgcn_{strides}")
    assert torch.allclose(c["one"], A.mstgcn(c["sd"], c["X"], eiu, 2, strides), rtol=1e-6, atol=1e-6)  # ARPACK seed
    assert torch.allclose(c["list"], A.mstgcn(c["sd"], c["X"], [eiu] * 6, 2, strides), rtol=1e-6, atol=1e-6)
