"""Golden values for EvolveGCNO / EvolveGCNH from the UNMODIFIED reference modules nn/recurrent/evolvegcno.py and evolvegcnh.py (imported
through oracle/refload.py, with the PyG pieces of tests/evolvegcn_seq.reference_classes), computed in float64.  Run in the build container
only:   python tests/golden/make_goldens_evolvegcn.py

Cases (tests/evolvegcn_seq.run: cumulative MSE / S, one backward per epoch, the weight detached between epochs; every parameter's
gradient, initial_weight and the pooling weight included):
* o_tutorial, h_tutorial      EvolveGCNO(4) / EvolveGCNH(20, 4) over the 103 chickenpox training snapshots, exactly as the examples
* o_two_epochs, h_two_epochs  the same over two epochs with `weight.detach()` between them
* o_raw                       EvolveGCNO(4, normalize=False) (the raw edge weights)
* h_improved                  EvolveGCNH(20, 4, improved=True)
* o_no_loops                  EvolveGCNO(4, add_self_loops=False)
* h_no_weight                 EvolveGCNH(20, 4) with edge_weight None
* o_wikimaths, h_wikimaths    C = 14 over the WikiMaths snapshots of gconvgru_wikimaths.pt.gz (1 068 nodes, weighted edges)
* o_unit, h_unit              the reference's unit-test shape: 100 nodes, C = 8, a seeded random weighted graph, 5 snapshots
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
from evolvegcn_seq import FIXTURE, RecurrentEGCN, fingerprint, graph_of, make_recurrent, reference_classes, run, seeded_state  # noqa: E402

OUT = os.path.join(HERE, FIXTURE)
D = torch.float64

# name: (kind, graph, C, nodes, epochs, normalize, improved, add_self_loops, edge weights, seed)
CASES = {
    "o_tutorial": ("O", "chickenpox", 4, 20, 1, True, False, True, True, 301),
    "h_tutorial": ("H", "chickenpox", 4, 20, 1, True, False, True, True, 302),
    "o_two_epochs": ("O", "chickenpox", 4, 20, 2, True, False, True, True, 303),
    "h_two_epochs": ("H", "chickenpox", 4, 20, 2, True, False, True, True, 304),
    "o_raw": ("O", "chickenpox", 4, 20, 1, False, False, True, True, 305),
    "h_improved": ("H", "chickenpox", 4, 20, 1, True, True, True, True, 306),
    "o_no_loops": ("O", "chickenpox", 4, 20, 1, True, False, False, True, 307),
    "h_no_weight": ("H", "chickenpox", 4, 20, 1, True, False, True, False, 308),
    "o_wikimaths": ("O", "wikimaths", 14, 1068, 1, True, False, True, True, 309),
    "h_wikimaths": ("H", "wikimaths", 14, 1068, 1, True, False, True, True, 310),
    "o_unit": ("O", "unit", 8, 100, 1, True, False, True, True, 311),
    "h_unit": ("H", "unit", 8, 100, 1, True, False, True, True, 312),
}


def describe(name):
    kind, graph, C, nodes, epochs, normalize, improved, loops, weights, seed = CASES[name]
    return dict(kind=kind, graph=graph, C=C, nodes=nodes, epochs=epochs, normalize=normalize, improved=improved, loops=loops,
                weights=weights, seed=seed)


def _case(classes, name):
    c = describe(name)
    ei, ew, X, Y = graph_of(c, HERE)
    m = RecurrentEGCN(make_recurrent(*classes, c), c["C"])
    m.load_state_dict({k: v.double() for k, v in seeded_state(c).items()})
    m = m.to(D)
    outs, cost = run(m, X.to(D), Y.to(D), ei, None if ew is None else ew.to(D), c["epochs"], retain=True)
    c.update(cost=cost.detach(), fingerprints={"out": fingerprint(outs), **{f"grad/{k}": fingerprint(p.grad) for k, p in m.named_parameters()}})
    return c


def main():
    classes = reference_classes()
    torch.set_default_dtype(D)
    cases = {name: _case(classes, name) for name in CASES}
    for k, c in cases.items():
        print(f"{k}: cost {float(c['cost']):.6f}")
    buf = io.BytesIO()
    torch.save(dict(cases=cases), buf)
    with gzip.GzipFile(OUT, "wb", compresslevel=9, mtime=0) as f:
        f.write(buf.getvalue())
    print(f"{os.path.basename(OUT)}  {os.path.getsize(OUT) / 1024:.0f} KB")


if __name__ == "__main__":
    main()
