"""Golden vectors for GConvGRU at 64 hidden channels, from the UNMODIFIED reference module (imported through oracle/refload.py, as
make_goldens_wikimaths.py does), computed in float64 and stored
rounded to float32 (costs in float64).  Run in the build container only:   python tests/golden/make_goldens_gconvgru64.py

It reuses the WikiMaths graph and series stored in gconvgru_wikimaths.pt.gz and the in-tree chickenpox data, so the fixture holds only the
parameters, predictions, costs and gradients of these cases (biases set to non-zero values), the tutorial model at 64 channels --
GConvGRU(F, 64, K), ReLU, Linear(64, 1):
* K2_sym, K1_sym  WikiMaths, H = None, cost_t = mean((y_hat.squeeze() - y_t)^2), one backward per snapshot, parameters fixed
* K2_rw           the same with normalization = "rw" and lambda_max = 1.6
* K2_sym_carried  H carried from a leaf H0 (tests/gconvgru64_seq.py's carried_h0), mean cost, one backward; plus dL/dH0
* chickenpox      GConvGRU(4, 64, 2) over the chickenpox training split: H = None per snapshot, the mean of the cumulative MSE, one backward
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
from gconvgru64_seq import RecurrentGCN64, carried_h0, run_chickenpox, run_wikimaths  # noqa: E402
from gconvgru_seq import chickenpox_train_split  # noqa: E402
from wikimaths_seq import load as load_wikimaths  # noqa: E402

OUT = os.path.join(HERE, "gconvgru64.pt.gz")
D = torch.float64
_STATES = {}


def _model(F, K, normalization, seed):
    gru = refload.load("nn.recurrent.gconv_gru")
    torch.manual_seed(seed)
    m = RecurrentGCN64(F, K, normalization, gru=gru.GConvGRU)
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for n_, p in m.named_parameters():
            if n_.endswith("bias"):
                p.copy_(torch.randn(p.shape, generator=g) * 0.1)
            p.copy_(p.float())                  # float32 values, as the models under test hold them
    state = _STATES.setdefault((F, K, seed), {k: v.detach().float().clone() for k, v in m.state_dict().items()})   # stored once
    assert all(torch.equal(v.double(), m.state_dict()[k]) for k, v in state.items())
    return m, state


def _grads(m):
    return {k: p.grad.detach().float() for k, p in m.named_parameters()}      # float64 sums, stored rounded to float32


def wiki_case(g, K, normalization="sym", lambda_max=None, carried=False, seed=0):
    m, state = _model(14, K, normalization, seed)
    ei, ew, X, Y = g["edge_index"], g["edge_weight"].to(D), g["X"].to(D), g["Y"].to(D)
    lam = None if lambda_max is None else torch.tensor(lambda_max, dtype=D)
    H0 = carried_h0(X.shape[1]).to(D).requires_grad_(True) if carried else None
    out, losses = run_wikimaths(m, X, Y, ei, ew, lam, H0)
    c = dict(K=K, normalization=normalization, lambda_max=None if lambda_max is None else torch.tensor(lambda_max), state=state,
             out=out.float(), losses=losses, grads=_grads(m))
    if carried:
        c.update(gH0=H0.grad.float())
    return c


def chickenpox_case(seed=43):
    m, state = _model(4, 2, "sym", seed)
    ei, ew, X, Y = chickenpox_train_split()
    out, cost = run_chickenpox(m, X.to(D), Y.to(D), ei, ew.to(D))
    cost.backward()
    return dict(K=2, normalization="sym", lambda_max=None, state=state, out=out.float(), cost=cost.detach(), grads=_grads(m))


def main():
    g = load_wikimaths(HERE)
    torch.set_default_dtype(D)                  # the reference builds its zero state with the default dtype
    cases = {"K2_sym": wiki_case(g, 2, seed=51), "K1_sym": wiki_case(g, 1, seed=52), "K2_rw": wiki_case(g, 2, "rw", 1.6, seed=51),
             "K2_sym_carried": wiki_case(g, 2, carried=True, seed=51), "chickenpox": chickenpox_case()}
    buf = io.BytesIO()
    torch.save(dict(cases=cases), buf)
    with gzip.GzipFile(OUT, "wb", compresslevel=9, mtime=0) as f:
        f.write(buf.getvalue())
    print(f"{os.path.basename(OUT)}  {os.path.getsize(OUT) / 1024:.0f} KB")


if __name__ == "__main__":
    main()
