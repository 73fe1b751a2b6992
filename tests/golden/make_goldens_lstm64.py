"""Golden values for GConvLSTM and GCLSTM at 64 hidden channels, from the UNMODIFIED reference modules (imported through oracle/refload.py,
as make_goldens_gconvgru64.py does), computed in float64.  Run in the build container only:   python tests/golden/make_goldens_lstm64.py

Each case's parameters come from its seed (tests/lstm64_seq.seeded_state), and the WikiMaths graph and series from gconvgru_wikimaths.pt.gz
and the in-tree chickenpox data, so the fixture holds only each case's description, the reference's cost and the fingerprints
(tests/lstm64_seq.fingerprint) of every prediction and gradient, for both modules, with tests/lstm64_seq.py's loop (H and C carried,
cumulative MSE / S, one backward):
* <module>/K2_sym, <module>/K1_sym  (14, 64, K) over the 6 WikiMaths snapshots, H and C carried from None
* <module>/K2_rw                    the same with normalization = "rw" and lambda_max = 1.6
* <module>/K2_sym_carried           H and C carried from leaf H0 / C0 (tests/lstm64_seq.carried_state); plus dL/dH0 and dL/dC0
* <module>/chickenpox               (4, 64, 2) over the chickenpox training split, H and C carried from None
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
from lstm64_seq import FIXTURE, RecurrentGCN64, carried_state, fingerprint, run, seeded_state  # noqa: E402
from gconvgru_seq import chickenpox_train_split  # noqa: E402
from wikimaths_seq import load as load_wikimaths  # noqa: E402

OUT = os.path.join(HERE, FIXTURE)
D = torch.float64
REF = {"gconv_lstm": ("nn.recurrent.gconv_lstm", "GConvLSTM"), "gc_lstm": ("nn.recurrent.gc_lstm", "GCLSTM")}


def _case(module, F, K, normalization, lambda_max, seed, X, Y, ei, ew, carried=False):
    path, name = REF[module]
    m = RecurrentGCN64(getattr(refload.load(path), name), F, K, normalization)
    m.load_state_dict({k: v.double() for k, v in seeded_state(module, F, K, seed).items()})
    m = m.to(D)
    n = X.shape[1]
    H0 = carried_state(n, 7, 13, 17).to(D).requires_grad_(True) if carried else None
    C0 = carried_state(n, 5, 11, 19).to(D).requires_grad_(True) if carried else None
    lam = None if lambda_max is None else torch.tensor(lambda_max, dtype=D)
    out, cost = run(m, X.to(D), Y.to(D), ei, ew.to(D), lam, H0, C0)
    cost.backward()
    fp = {"out": fingerprint(out), **{f"grad/{k}": fingerprint(p.grad) for k, p in m.named_parameters()}}
    if carried:
        fp.update(gH0=fingerprint(H0.grad), gC0=fingerprint(C0.grad))
    return dict(module=module, F=F, K=K, normalization=normalization, seed=seed,
                lambda_max=None if lambda_max is None else torch.tensor(lambda_max), cost=cost.detach(), fingerprints=fp)


def main():
    g = load_wikimaths(HERE)
    torch.set_default_dtype(D)                  # the reference builds its zero states with the default dtype
    ei, ew, X, Y = g["edge_index"], g["edge_weight"], g["X"], g["Y"]
    cei, cew, cX, cY = chickenpox_train_split()
    cases = {}
    for i, module in enumerate(REF):
        s = 61 + 10 * i
        for key, K, norm, lam, carried, seed in (("K2_sym", 2, "sym", None, False, s), ("K1_sym", 1, "sym", None, False, s + 1),
                                                 ("K2_rw", 2, "rw", 1.6, False, s), ("K2_sym_carried", 2, "sym", None, True, s)):
            cases[f"{module}/{key}"] = _case(module, 14, K, norm, lam, seed, X, Y, ei, ew, carried)
        cases[f"{module}/chickenpox"] = _case(module, 4, 2, "sym", None, s + 5, cX, cY, cei, cew)
    for k, c in cases.items():
        print(f"{k}: cost {float(c['cost']):.6f}")
    buf = io.BytesIO()
    torch.save(dict(cases=cases), buf)
    with gzip.GzipFile(OUT, "wb", compresslevel=9, mtime=0) as f:
        f.write(buf.getvalue())
    print(f"{os.path.basename(OUT)}  {os.path.getsize(OUT) / 1024:.0f} KB")


if __name__ == "__main__":
    main()
