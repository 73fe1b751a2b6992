"""Golden values for LRGCN from the UNMODIFIED reference module nn/recurrent/lrgcn.py (imported through oracle/refload.py, with
torch_geometric.nn.RGCNConv provided by tests/lrgcn_seq.RGCNConv, the restated per-relation loop), computed in float64.  Run in the build
container only:   python tests/golden/make_goldens_lrgcn.py

Cases (tests/lrgcn_seq.run: H and C carried, cumulative MSE / S, one backward):
* tutorial            LRGCN(4, 32, 1, 1) over the 103 chickenpox training snapshots with the float edge_attr as edge_type, exactly as
                      examples/recurrent/lrgcn_example.py writes it: no edge has type 0, so weight / comp get exactly zero gradients
* chickenpox_R1_B1, chickenpox_R1_None   the same with integer types, all 0
* chickenpox_R2_B1, chickenpox_R2_None   R = 2 with edge_type = (src < dst)
* wikimaths_32_R2_B2[_carried]           LRGCN(14, 32, 2, 2) over the WikiMaths snapshots of gconvgru_wikimaths.pt.gz, types (src < dst)
* wikimaths_64_R1_B1[_carried]           LRGCN(14, 64, 1, 1), all types 0; _carried: H and C from leaf H0 / C0, plus dL/dH0, dL/dC0
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
from lrgcn_seq import FIXTURE, RGCNConv, RecurrentLRGCN, edge_types, fingerprint, run, seeded_state, states_for  # noqa: E402
from gconvgru_seq import chickenpox_train_split  # noqa: E402
from wikimaths_seq import load as load_wikimaths  # noqa: E402

OUT = os.path.join(HERE, FIXTURE)
D = torch.float64


def _reference_lrgcn():
    sys.path.insert(0, refload._STUBS)
    import torch_geometric.nn as tgnn
    tgnn.RGCNConv = RGCNConv
    return refload.load("nn.recurrent.lrgcn").LRGCN


def _case(cls, graph, F, out, R, B, types, seed, carried=False):
    ei, ew, X, Y = graph
    c = dict(graph="chickenpox" if F == 4 else "wikimaths", F=F, out=out, R=R, B=B, types=types, seed=seed, carried=carried)
    m = RecurrentLRGCN(cls, F, out, R, B)
    m.load_state_dict({k: v.double() for k, v in seeded_state(c).items()})
    m = m.to(D)
    H0, C0 = states_for(c, X.shape[1], dtype=D)
    et = edge_types(types, ei, ew.to(D) if types == "attr" else ew)
    outs, cost = run(m, X.to(D), Y.to(D), ei, et, H0, C0)
    cost.backward()
    fp = {"out": fingerprint(outs), **{f"grad/{k}": fingerprint(p.grad) for k, p in m.named_parameters()}}
    if carried:
        fp.update(gH0=fingerprint(H0.grad), gC0=fingerprint(C0.grad))
    c.update(cost=cost.detach(), fingerprints=fp)
    return c


def main():
    cls = _reference_lrgcn()
    torch.set_default_dtype(D)                  # the reference builds its zero states with the default dtype
    g = load_wikimaths(HERE)
    wiki = (g["edge_index"], g["edge_weight"], g["X"], g["Y"])
    pox = chickenpox_train_split()
    cases = {"tutorial": _case(cls, pox, 4, 32, 1, 1, "attr", 101)}
    for R, types in ((1, "zero"), (2, "src_lt_dst")):
        for B in (1, None):
            cases[f"chickenpox_R{R}_B{B}"] = _case(cls, pox, 4, 32, R, B, types, 110 + 10 * R + (B or 0))
    for carried in (False, True):
        sfx = "_carried" if carried else ""
        cases[f"wikimaths_32_R2_B2{sfx}"] = _case(cls, wiki, 14, 32, 2, 2, "src_lt_dst", 141, carried)
        cases[f"wikimaths_64_R1_B1{sfx}"] = _case(cls, wiki, 14, 64, 1, 1, "zero", 151, carried)
    for k, c in cases.items():
        print(f"{k}: cost {float(c['cost']):.6f}")
    buf = io.BytesIO()
    torch.save(dict(cases=cases), buf)
    with gzip.GzipFile(OUT, "wb", compresslevel=9, mtime=0) as f:
        f.write(buf.getvalue())
    print(f"{os.path.basename(OUT)}  {os.path.getsize(OUT) / 1024:.0f} KB")


if __name__ == "__main__":
    main()
