"""Golden values for HeteroGCLSTM from the UNMODIFIED reference module nn/hetero/heterogclstm.py (imported through oracle/refload.py on
oracle/stubs, with tests/hetero_gclstm_seq.py's restated SAGEConv / HeteroConv installed), computed in float64 on the CPU.  Run in the
build container only:   python tests/golden/make_goldens_hetero_gclstm.py

Cases (tests/hetero_gclstm_seq.CASES): the loss, and the float64 fingerprints (tests/lstm64_seq.fingerprint) of every output and every
gradient (X's or H0 / C0's and each parameter's).
Parameters are not stored: they come from the case's seed (construction, then the reference's first-forward materialisation)."""
import gzip
import io
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
from hetero_gclstm_seq import CASES, FIXTURE, build, fingerprint, materialize_reference, reference_class, run  # noqa: E402
from pytorch_geometric_temporal_b200.signal import StaticHeteroGraphTemporalSignal  # noqa: E402

OUT = os.path.join(HERE, FIXTURE)


def main():
    torch.set_default_dtype(torch.float64)
    cls = reference_class()
    cases = {}
    for name, case in CASES.items():
        m, inputs, metadata, _ = build(cls, case)
        materialize_reference(m, inputs, metadata)
        outs, grads, loss = run(m, case, inputs, metadata, "cpu", torch.float64, StaticHeteroGraphTemporalSignal)
        cases[name] = dict(case, loss=loss, fingerprints={k: fingerprint(v) for k, v in {**outs, **{f'grad.{g}': v for g, v in grads.items()}}.items()})
        print(f"{name}: loss {float(loss):.6f}, {len(outs)} outputs, {len(grads)} gradients")
    buf = io.BytesIO()
    torch.save(dict(cases=cases), buf)
    with gzip.GzipFile(OUT, "wb", compresslevel=9, mtime=0) as f:
        f.write(buf.getvalue())
    print(f"{os.path.basename(OUT)}  {os.path.getsize(OUT) / 1024:.0f} KB")


if __name__ == "__main__":
    main()
