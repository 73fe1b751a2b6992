"""Golden values for AGCRN from the UNMODIFIED reference module nn/recurrent/agcrn.py (imported through oracle/refload.py on oracle/stubs),
computed in float64.  Run in the build container only:   python tests/golden/make_goldens_agcrn.py

Cases (tests/agcrn_seq.CASES, one forward and backward each): the output, the cost and every gradient (the parameters', E's when it is
trained, X's for the unit and paper cases) as float64 fingerprints, and those of at most 16 384 elements also as float32 roundings
of the float64 values (2^-24 relative, far below the tests' 2^-20 floor):
* tutorial        the example's epoch: AGCRN(20, 8, 2, 2, 4), ReLU, Linear(2, 1), 102 chickenpox snapshots at lags 8, h carried, E fixed
* tutorial_e      the same with E a trained parameter
* k1, k3          the same at K = 1 (the single weight block on Y + S Y) and K = 3 (T_2 = 2 S S - I)
* unit_k2/_k3     the reference's unit-test shape: N = 100, in 64, out 16, d 32, H carried into a second call
* paper           the paper's two stacked layers (1 -> 64, 64 -> 64), d = 10, K = 2, 307 nodes, B = 4, T = 12
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
from agcrn_seq import CASES, FIXTURE, fingerprint, model_for, reference_class, run  # noqa: E402

OUT = os.path.join(HERE, FIXTURE)
D = torch.float64


def _case(name):
    c = dict(CASES[name])
    m = model_for(c, reference_class(), "cpu", D)
    out, cost, grads = run(m, c, "cpu", D)
    got = dict(out=out, **{f"grad.{k}": v for k, v in grads.items()})
    c.update(cost=cost, values={k: v.float() for k, v in got.items() if v.numel() <= 16384},
             fingerprints={k: fingerprint(v) for k, v in got.items()})
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
