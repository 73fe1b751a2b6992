"""Golden vectors for ASTGCN on graphs wider than one spatial-attention row tile (> 320 nodes), from the UNMODIFIED reference module
(imported through oracle/refload.py on top of oracle/stubs).  Run in the build container only:
python tests/golden/make_goldens_astgcn_large.py

astgcn_large.pt.gz -- ASTGCN(3 blocks, K=3, 64/64 filters, stride 1, 12 -> 12), the cfg4 architecture, on
  * pems07_sym  : the PeMS07-shaped graph (883 nodes, 866 links), normalization "sym"
  * pems07_none : the same graph, normalization None (lambda_max by scipy, as the reference computes it)
  * pems03_sym  : the PeMS03-shaped graph (358 nodes, 547 links), normalization "sym"
Each case holds the graph, the parameter seed (the module is built under torch.manual_seed(seed): Vs / bs alone are 3 x 2 x N x N floats,
so the tests rebuild the parameters instead of reading them) with a checksum of the parameters, the input seed, X (B windows) and the
output.  The reference runs in float64 on the float32 parameters and inputs and the output is stored in float32, so the golden holds the
exact values and a test measures the error of the path under test alone.
"""
import gzip
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import refload  # noqa: E402
from pytorch_geometric_temporal_b200.dataset import synthetic  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "astgcn_large.pt.gz")
CTOR = dict(nb_block=3, in_channels=1, K=3, nb_chev_filter=64, nb_time_filter=64, time_strides=1, num_for_predict=12, len_input=12)
GRAPHS = {"pems07": (synthetic.pems07_like, 883), "pems03": (synthetic.pems03_like, 358)}
CASES = {"pems07_sym": ("pems07", "sym", 0, 21, 4), "pems07_none": ("pems07", None, 1, 22, 3), "pems03_sym": ("pems03", "sym", 2, 23, 4)}


def make_case(mod, graph, norm, seed, x_seed, B):
    like, n = GRAPHS[graph]
    eiu = torch.from_numpy(like(0))
    torch.manual_seed(seed)
    m = mod.ASTGCN(**CTOR, num_of_vertices=n, normalization=norm)
    checksum = float(sum(v.double().abs().sum() for v in m.state_dict().values()))
    X = torch.randn(B, n, 1, 12, generator=torch.Generator().manual_seed(x_seed))
    with torch.no_grad():
        out32 = m(X, eiu)
        old = torch.get_default_dtype()
        torch.set_default_dtype(torch.float64)
        try:
            out = m.double()(X.double(), eiu)
        finally:
            torch.set_default_dtype(old)
    err32 = (out32.double() - out).abs().max().item()
    print(f"  {graph} {norm}: |out| max {out.abs().max().item():.3f}, float32 reference vs float64 max abs err {err32:.2e}")
    return dict(graph=graph, graph_seed=0, edge_index=eiu, normalization=norm, seed=seed, state_checksum=checksum, x_seed=x_seed, X=X,
                out=out.float())


def main():
    mod = refload.load("nn.attention.astgcn")
    cases = {name: make_case(mod, *spec) for name, spec in CASES.items()}
    with gzip.open(OUT, "wb", compresslevel=9) as f:
        torch.save(dict(ctor=CTOR, cases=cases), f)
    print(f"astgcn_large.pt.gz  {os.path.getsize(OUT) / 1024:.0f} KB")


if __name__ == "__main__":
    main()
