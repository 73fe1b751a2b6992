"""Golden values for MTGNN from the UNMODIFIED reference module nn/attention/mtgnn.py (imported through oracle/refload.py; it imports
only torch), computed in float64 on the CPU.  Run in the build container only:   python tests/golden/make_goldens_mtgnn.py

Cases: tests/mtgnn_seq.CASES.  For each, every output, loss and parameter gradient of the two training steps and the eval output
(tests/mtgnn_seq.run) as a float64 fingerprint, stacked into one (keys, 5) tensor with its key list; the losses also as values.
Every learned graph the run builds must keep a gap of at least 2^-20 (relative) between the k-th and (k+1)-th values of each row
whose k-th value is positive, so that float32 cannot select another set; the script fails otherwise (re-seed the case)."""
import gzip
import io
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
from mtgnn_seq import CASES, FIXTURE, fingerprint, model_for, reference_module, run  # noqa: E402

OUT = os.path.join(HERE, FIXTURE)
D = torch.float64
GAP = 2.0 ** -20


@torch.no_grad()
def min_gap(mod, idx, FE):
    """The smallest relative gap between the k-th and (k+1)-th values over the rows of the graph mod builds, before its mask."""
    if FE is None:
        v1, v2 = mod._embedding1(idx), mod._embedding2(idx)
    else:
        v1 = v2 = FE[idx, :]
    v1, v2 = torch.tanh(mod._alpha * mod._linear1(v1)), torch.tanh(mod._alpha * mod._linear2(v2))
    A = torch.relu(torch.tanh(mod._alpha * (v1 @ v2.T - v2 @ v1.T))).detach()
    top = A.topk(min(mod._k + 1, A.shape[1]), 1).values
    if top.shape[1] <= mod._k:
        return float("inf")
    kth, nxt = top[:, mod._k - 1], top[:, mod._k]
    live = kth > 0
    return float(((kth - nxt) / kth)[live].min()) if live.any() else float("inf")


def _case(name):
    c = dict(CASES[name])
    gaps = []
    ref = reference_module()
    got = run(model_for(c, ref.MTGNN, "cpu", D), c, "cpu", D, on_graph=lambda mod, idx, FE: gaps.append(min_gap(mod, idx, FE)))
    gap = min(gaps, default=float("inf"))
    assert gap >= GAP, f"{name}: a learned graph row has a top-k gap of {gap:.3g} < 2^-20: re-seed the case"
    c.update(values={k: v.float() for k, v in got.items() if k.startswith("loss.")}, min_gap=gap,
             fingerprint_keys=list(got), fingerprints=torch.stack([fingerprint(v) for v in got.values()]))
    return c


def main():
    torch.set_default_dtype(D)         # the reference builds its masks and identity in the default dtype
    cases = {name: _case(name) for name in CASES}
    for k, c in cases.items():
        print(f"{k}: loss {float(c['values']['loss.0']):.6f}  min top-k gap {c['min_gap']:.3g}")
    buf = io.BytesIO()
    torch.save(dict(cases=cases), buf)
    with gzip.GzipFile(OUT, "wb", compresslevel=9, mtime=0) as f:
        f.write(buf.getvalue())
    print(f"{os.path.basename(OUT)}  {os.path.getsize(OUT) / 1024:.0f} KB")


if __name__ == "__main__":
    main()
