"""Golden values for DyGrEncoder from the UNMODIFIED reference module nn/recurrent/dygrae.py (imported through oracle/refload.py, with
torch_geometric.nn.GatedGraphConv provided by tests/dygrae_seq.GatedGraphConv, the restated PyG 2.x layer), computed in float64.  Run in
the build container only:   python tests/golden/make_goldens_dygrae.py

Cases (tests/dygrae_seq.run: cumulative MSE / S, one backward; `state` "carry": H and C carried from None, "leaf": carried from leaf H0 /
C0 with dL/dH0 and dL/dC0, "none": None at every snapshot):
* tutorial               DyGrEncoder(4, 1, "mean", 32, 1) over the 103 chickenpox training snapshots, edge weights the example's edge_attr
                         (ones), exactly as examples/recurrent/dygrencoder_example.py writes it
* tutorial_add, tutorial_max           the same with "add" and "max"
* chickenpox_max_3_64    DyGrEncoder(4, 3, "max", 64, 1) on chickenpox
* chickenpox_add_leaf    DyGrEncoder(4, 2, "add", 32, 1) on chickenpox from leaf H0 / C0
* wikimaths_max_16_64    DyGrEncoder(16, 2, "max", 64, 1) over the WikiMaths snapshots of gconvgru_wikimaths.pt.gz (weighted edges)
* wikimaths_mean_32_32   DyGrEncoder(32, 2, "mean", 32, 1) (C > 16: the cuDNN LSTM stage)
* wikimaths_add_lstm2    DyGrEncoder(16, 1, "add", 32, 2) with H = C = None at every snapshot
"""
import gzip
import io
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
from oracle import refload  # noqa: E402
from dygrae_seq import FIXTURE, GatedGraphConv, RecurrentDyGr, fingerprint, run, seeded_state, states_for  # noqa: E402
from gconvgru_seq import chickenpox_train_split  # noqa: E402
from wikimaths_seq import load as load_wikimaths  # noqa: E402

OUT = os.path.join(HERE, FIXTURE)
D = torch.float64

CASES = {
    "tutorial": ("chickenpox", 4, 1, "mean", 32, 1, "carry", 201),
    "tutorial_add": ("chickenpox", 4, 1, "add", 32, 1, "carry", 202),
    "tutorial_max": ("chickenpox", 4, 1, "max", 32, 1, "carry", 203),
    "chickenpox_max_3_64": ("chickenpox", 4, 3, "max", 64, 1, "carry", 204),
    "chickenpox_add_leaf": ("chickenpox", 4, 2, "add", 32, 1, "leaf", 205),
    "wikimaths_max_16_64": ("wikimaths", 16, 2, "max", 64, 1, "carry", 206),
    "wikimaths_mean_32_32": ("wikimaths", 32, 2, "mean", 32, 1, "carry", 207),
    "wikimaths_add_lstm2": ("wikimaths", 16, 1, "add", 32, 2, "none", 208),
}


def describe(name):
    graph, C, Lg, aggr, Ho, Ll, state, seed = CASES[name]
    return dict(graph=graph, C=C, Lg=Lg, aggr=aggr, Ho=Ho, Ll=Ll, state=state, seed=seed)


def _reference_dygrae():
    sys.path.insert(0, refload._STUBS)
    import torch_geometric.nn as tgnn
    tgnn.GatedGraphConv = GatedGraphConv
    return refload.load("nn.recurrent.dygrae").DyGrEncoder


def _case(cls, graphs, name):
    c = describe(name)
    ei, ew, X, Y = graphs[c["graph"]]
    m = RecurrentDyGr(cls, c["C"], c["Lg"], c["aggr"], c["Ho"], c["Ll"])
    m.load_state_dict({k: v.double() for k, v in seeded_state(c).items()})
    m = m.to(D)
    H0, C0 = states_for(c, X.shape[1], dtype=D)
    outs, cost = run(m, X.to(D), Y.to(D), ei, ew.to(D), H0, C0, c["state"] != "none")
    cost.backward()
    fp = {"out": fingerprint(outs), **{f"grad/{k}": fingerprint(p.grad) for k, p in m.named_parameters()}}
    if H0 is not None:
        fp.update(gH0=fingerprint(H0.grad), gC0=fingerprint(C0.grad))
    c.update(cost=cost.detach(), fingerprints=fp)
    return c


def main():
    cls = _reference_dygrae()
    torch.set_default_dtype(D)
    g = load_wikimaths(HERE)
    graphs = {"chickenpox": chickenpox_train_split(), "wikimaths": (g["edge_index"], g["edge_weight"], g["X"], g["Y"])}
    cases = {name: _case(cls, graphs, name) for name in CASES}
    for k, c in cases.items():
        print(f"{k}: cost {float(c['cost']):.6f}")
    buf = io.BytesIO()
    torch.save(dict(cases=cases), buf)
    with gzip.GzipFile(OUT, "wb", compresslevel=9, mtime=0) as f:
        f.write(buf.getvalue())
    print(f"{os.path.basename(OUT)}  {os.path.getsize(OUT) / 1024:.0f} KB")


if __name__ == "__main__":
    main()
