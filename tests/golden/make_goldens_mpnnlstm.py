"""Golden values for MPNNLSTM from the UNMODIFIED reference module nn/recurrent/mpnn_lstm.py (imported through oracle/refload.py on
oracle/stubs, its dropout given the masks of tests/mpnnlstm_seq.Masks through a replaced F), computed in float64.  Run in the build
container only:   python tests/golden/make_goldens_mpnnlstm.py

Cases (tests/mpnnlstm_seq.run: cumulative MSE / S and one backward per epoch in training mode; the outputs, the cost, every parameter's
gradient and BatchNorm's running statistics recorded):
* tutorial        MPNNLSTM(4, 32, 20, 1, 0.5), ReLU, Linear(68, 1) over the 103 chickenpox training snapshots, exactly as the example
* two_epochs      the same over two epochs (num_batches_tracked = 206), then an eval pass over the test split
* p0              dropout 0
* momentum_none   both BatchNorms with momentum=None (the cumulative average)
* no_weight       edge_weight None
* window4         MPNNLSTM(1, 32, 20, 4, 0.5) on chickenpox's four lags as 80 x 1 rows
* window2_b2      MPNNLSTM(4, 32, 20, 2, 0.5) on B = 2 windows of 2 snapshots (80 rows; only the first 20 see the graph's edges)
* unit            the reference's unit-test shape: 100 nodes, in_channels 64, a seeded random weighted graph, 5 snapshots
* wikimaths       MPNNLSTM(14, 32, 1068, 1, 0.5) over the WikiMaths snapshots of gconvgru_wikimaths.pt.gz
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
from mpnnlstm_seq import FIXTURE, Masks, fingerprint, graph_of, make, reference_class, results, run, seeded_state  # noqa: E402

OUT = os.path.join(HERE, FIXTURE)
D = torch.float64

# name: (graph, cin, nodes, window, p, epochs, eval, momentum, edge weights, seed)
CASES = {
    "tutorial": ("chickenpox", 4, 20, 1, 0.5, 1, False, "default", True, 401),
    "two_epochs": ("chickenpox", 4, 20, 1, 0.5, 2, True, "default", True, 402),
    "p0": ("chickenpox", 4, 20, 1, 0.0, 1, False, "default", True, 403),
    "momentum_none": ("chickenpox", 4, 20, 1, 0.5, 1, False, None, True, 404),
    "no_weight": ("chickenpox", 4, 20, 1, 0.5, 1, False, "default", False, 405),
    "window4": ("chickenpox", 1, 20, 4, 0.5, 1, False, "default", True, 406),
    "window2_b2": ("chickenpox", 4, 20, 2, 0.5, 1, False, "default", True, 407),
    "unit": ("unit", 64, 100, 1, 0.5, 1, False, "default", True, 408),
    "wikimaths": ("wikimaths", 14, 1068, 1, 0.5, 1, False, "default", True, 409),
}


def describe(name):
    graph, cin, nodes, window, p, epochs, ev, momentum, weights, seed = CASES[name]
    return dict(graph=graph, cin=cin, nodes=nodes, window=window, p=p, epochs=epochs, eval=ev, momentum=momentum, weights=weights, seed=seed)


def _case(name):
    c = describe(name)
    ei, ew, train, ev = graph_of(c, HERE)
    m = make(reference_class(Masks(c["seed"])), c)
    m.load_state_dict(seeded_state(c))
    m = m.to(D)
    dd = lambda xy: None if xy is None else (xy[0].to(D), xy[1].to(D))
    outs, cost, evs = run(m, dd(train), dd(ev), ei, None if ew is None else ew.to(D), c["epochs"], retain=True)
    got = results(outs.detach(), cost, evs, {k: p.grad for k, p in m.named_parameters()},
                  {k: v for k, v in m.state_dict().items() if "running" in k or "num_batches" in k})
    c.update(cost=cost.detach(), fingerprints={k: fingerprint(v) for k, v in got.items()})
    return c


def main():
    torch.set_default_dtype(D)
    cases = {name: _case(name) for name in CASES}
    for k, c in cases.items():
        print(f"{k}: cost {float(c['cost']):.6f}")
    buf = io.BytesIO()
    torch.save(dict(cases=cases), buf)
    with gzip.GzipFile(OUT, "wb", compresslevel=9, mtime=0) as f:
        f.write(buf.getvalue())
    print(f"{os.path.basename(OUT)}  {os.path.getsize(OUT) / 1024:.0f} KB")


if __name__ == "__main__":
    main()
