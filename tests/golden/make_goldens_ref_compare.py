"""Golden data for the tests that compare with the UNMODIFIED reference (tests/test_oracle_vs_reference.py, the loader and
dynamic-signal tests of tests/test_next_rows_cpu.py, the IndexDataset test of tests/test_signal.py).  The reference is imported
through oracle/refload.py on top of oracle/stubs, run on the inputs those tests use, and its outputs -- with the state dicts and
random inputs they depend on -- are written to ref_compare.pt.gz (host-side structures as digests, oracle/golden.py), so that
the tests need nothing outside the repository.
Run where the reference tree exists:  python tests/golden/make_goldens_ref_compare.py
"""
import gzip
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import attention as A, pyg, refload  # noqa: E402
from oracle.golden import PATH as OUT, digest  # noqa: E402


def sd(m):
    return {k: v.detach().clone() for k, v in m.state_dict().items()}


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


def oracle_cases():
    out = {}
    ei, ew = _graph()
    for K in (1, 2, 3, 4):
        m = refload.load("nn.recurrent.dcrnn")
        torch.manual_seed(K)
        ref = m.DCRNN(2, 8, K)
        X, H = torch.randn(12, 2), torch.randn(12, 8)
        with torch.no_grad():
            c = {"sd": sd(ref), "X": X, "H": H, "out_h": ref(X, ei, ew, H), "out": ref(X, ei)}
            refb = m.BatchedDCRNN(2, 8, K)
            Xb = torch.randn(3, 4, 12, 2)
            c.update(sdb=sd(refb), Xb=Xb, outb=refb(Xb, ei, ew))
        out[f"dcrnn_K{K}"] = c
    for K in (1, 2, 3, 4):
        for norm in ("sym", "rw", None):
            lm = None if norm == "sym" else torch.tensor(2.3)
            X, H, C = torch.randn(12, 4), torch.randn(12, 8), torch.randn(12, 8)
            with torch.no_grad():
                g = refload.load("nn.recurrent.gconv_gru").GConvGRU(4, 8, K, normalization=norm)
                l = refload.load("nn.recurrent.gconv_lstm").GConvLSTM(4, 8, K, normalization=norm)
                out[f"gconv_K{K}_{norm}"] = {"X": X, "H": H, "C": C, "sd_gru": sd(g), "gru": g(X, ei, ew, H, lm),
                                             "sd_lstm": sd(l), "lstm": l(X, ei, ew, H, C, lm)}
    m = refload.load("nn.recurrent.temporalgcn")
    a = refload.load("nn.recurrent.attentiontemporalgcn")
    X, H = torch.randn(12, 4), torch.randn(12, 8)
    c = {"X": X, "H": H}
    with torch.no_grad():
        for improved in (False, True):
            for asl in (True, False):
                ref = m.TGCN(4, 8, improved=improved, add_self_loops=asl)
                c[f"tgcn_{improved}_{asl}"] = (sd(ref), ref(X, ei, ew, H))
        ref = m.TGCN2(4, 8, 3)
        Xb, Hb = torch.randn(3, 12, 4), torch.randn(3, 12, 8)
        c.update(Xb=Xb, Hb=Hb, tgcn2=(sd(ref), ref(Xb, ei, ew, Hb)))
        ref = a.A3TGCN2(4, 8, 6, 3)
        Xp = torch.randn(3, 12, 4, 6)
        c.update(Xp=Xp, a3tgcn2=(sd(ref), ref(Xp, ei, ew)))
        ref = a.A3TGCN(4, 8, 6)
        c["a3tgcn"] = (sd(ref), ref(Xp[0], ei, ew))
    out["tgcn_family"] = c
    eiu = _undirected(ei)
    for norm in ("sym", None, "rw"):
        ref = refload.load("nn.attention.astgcn").ASTGCN(2, 1, 3, 8, 8, 2, 4, 6, 12, normalization=norm)
        Xa = torch.randn(3, 12, 1, 6)
        lm = None
        if norm != "sym":
            lm = pyg.LaplacianLambdaMax()(pyg.Data(edge_index=eiu, edge_attr=None, num_nodes=12)).lambda_max
        with torch.no_grad():
            out[f"astgcn_{norm}"] = {"sd": sd(ref), "X": Xa, "lm": lm, "want": ref(Xa, eiu)}
    for norm in ("sym", None, "rw"):
        torch.manual_seed(0)
        ref = refload.load("nn.attention.astgcn").ChebConvAttention(5, 7, K=3, normalization=norm)
        ei2 = torch.tensor([[0, 1, 1, 2, 3, 4, 5, 6, 3, 6], [1, 0, 2, 1, 4, 3, 6, 5, 6, 3]])
        ew2 = torch.rand(ei2.size(1)) + 0.1
        x, S = torch.randn(3, 7, 5), torch.softmax(torch.rand(3, 7, 7), dim=1)
        batch, lam = torch.tensor([0, 0, 0, 1, 1, 1, 1]), torch.tensor([2.0, 3.0])
        with torch.no_grad():
            out[f"chebatt_{norm}"] = {"sd": sd(ref), "ew": ew2, "x": x, "S": S, "want": ref(x, ei2, S, ew2, batch, lam),
                                      "want_one_lambda": ref(x, ei2, S, ew2, None, 2.0)}
    for K in (1, 2, 3):
        for norm in ("sym", "rw", None):
            lm = None if norm == "sym" else torch.tensor(2.3)
            X, H, C = torch.randn(12, 4), torch.randn(12, 8), torch.randn(12, 8)
            with torch.no_grad():
                ref = refload.load("nn.recurrent.gc_lstm").GCLSTM(4, 8, K, normalization=norm)
                out[f"gc_lstm_K{K}_{norm}"] = {"sd": sd(ref), "X": X, "H": H, "C": C, "full": ref(X, ei, ew, H, C, lm),
                                               "bare": ref(X, ei, lambda_max=lm)}
    for K in (1, 2, 3):
        ref = refload.load("nn.attention.stgcn").STConv(12, 3, 8, 6, 3, K)
        X = torch.randn(2, 9, 12, 3)
        with torch.no_grad():
            c = {"X": X, "sd_train": sd(ref)}
            c["train"] = ref(X, ei, ew)                      # module default: training-mode BatchNorm
            A.stconv(ref.state_dict(), X, ei, ew)            # what the test calls in between, on the module's own tensors
            ref.eval()
            c["sd_eval"] = sd(ref)
            c["eval"] = ref(X, ei, ew)
            c["tconv1"] = ref._temporal_conv1(X)
        out[f"stconv_K{K}"] = c
    for strides in (1, 2):
        ref = refload.load("nn.attention.mstgcn").MSTGCN(2, 2, 3, 8, 8, strides, 4, 6)
        X = torch.randn(3, 12, 2, 6)
        with torch.no_grad():
            out[f"mstgcn_{strides}"] = {"sd": sd(ref), "X": X, "one": ref(X, eiu), "list": ref(X, [eiu] * 6)}
    return out


def loader_cases():
    from test_next_rows_cpu import _archive
    out = {}
    for mod, name, prefix in (("dataset.metr_la", "METRLADatasetLoader", ""), ("dataset.pems_bay", "PemsBayDatasetLoader", "pems_")):
        with tempfile.TemporaryDirectory() as tmp:
            _archive(tmp, 9, 2, 60, prefix)
            open(os.path.join(tmp, "METR-LA.zip" if prefix == "" else "PEMS-BAY.zip"), "wb").close()
            sig = refload.load("signal.static_graph_temporal_signal")
            sys.modules["torch_geometric_temporal.signal"].StaticGraphTemporalSignal = sig.StaticGraphTemporalSignal
            ref_cls = getattr(refload.load(mod), name)
            want = ref_cls(raw_data_dir=tmp).get_dataset(6, 6)
            snaps = [tuple(digest(t) for t in (a.x, a.y, a.edge_index, a.edge_attr)) for a in want]
            w = ref_cls(raw_data_dir=tmp, index=True).get_index_dataset(lags=6, batch_size=4)
            loaders = [[(digest(xa), digest(ya)) for xa, ya in w[i]] for i in range(3)]
            rest = [digest(w[i]) for i in range(3, 7)]
            w = ref_cls(raw_data_dir=tmp, index=True).get_index_dataset(lags=6, batch_size=4, shuffle=True, world_size=2, ddp_rank=1)
            ddp = [(digest(xa), digest(ya)) for xa, ya in w[0]]
        out[name] = {"snapshots": snaps, "loaders": loaders, "rest": rest, "ddp_rank1": ddp}
    return out


def dynamic_cases():
    from test_next_rows_cpu import _dynamic_case
    eis, ews, xs, ys, bs, marks = _dynamic_case(seed=3)
    pairs = {
        "DynamicGraphTemporalSignal": (refload.load("signal.dynamic_graph_temporal_signal").DynamicGraphTemporalSignal, (eis, ews, xs, ys)),
        "DynamicGraphStaticSignal": (refload.load("signal.dynamic_graph_static_signal").DynamicGraphStaticSignal, (eis, ews, xs[0], ys)),
        "DynamicGraphTemporalSignalBatch": (refload.load("signal.dynamic_graph_temporal_signal_batch").DynamicGraphTemporalSignalBatch,
                                            (eis, ews, xs, ys, bs)),
        "DynamicGraphStaticSignalBatch": (refload.load("signal.dynamic_graph_static_signal_batch").DynamicGraphStaticSignalBatch,
                                          (eis, ews, xs[0], ys, bs)),
        "StaticGraphTemporalSignalBatch": (refload.load("signal.static_graph_temporal_signal_batch").StaticGraphTemporalSignalBatch,
                                           (eis[0], ews[0], xs, ys, bs[0])),
    }
    out = {}
    for name, (cls, args) in pairs.items():
        want = cls(*args, marks=marks)
        snaps = []
        for a in want:
            d = {k: digest(getattr(a, k)) for k in ("x", "edge_index", "edge_attr", "y", "marks")}
            d["batch"] = digest(getattr(a, "batch", None))
            snaps.append(d)
        wa = want[1:4]
        out[name] = {"count": want.snapshot_count, "snapshots": snaps, "slice_count": wa.snapshot_count, "slice_x0": digest(wa[0].x),
                     "slice_ei2": digest(wa[2].edge_index)}
    return out


def index_dataset_case():
    from pytorch_geometric_temporal_b200.signal import index_splits
    rng = np.random.RandomState(0)
    data = rng.rand(60, 7, 2).astype(np.float32)
    tr, _, _ = index_splits(60, 12)
    ref = refload.load("signal.index_dataset").IndexDataset(tr, data, 12)
    return [(digest(ref[i][0]), digest(ref[i][1])) for i in range(len(ref))]


if __name__ == "__main__":
    assert refload.available(), "needs the reference tree"
    data = {"oracle": oracle_cases(), "loaders": loader_cases(), "dynamic": dynamic_cases(), "index_dataset": index_dataset_case()}
    with gzip.GzipFile(OUT, "wb", compresslevel=9, mtime=0) as f:
        torch.save(data, f)
    print(f"{os.path.basename(OUT)}  {os.path.getsize(OUT) / 1024:.0f} KB")
