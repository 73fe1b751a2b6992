"""Golden values for GMAN from the UNMODIFIED reference module nn/attention/gman.py (imported through oracle/refload.py, no stubs
needed), computed in float64.  Run in the build container only:   python tests/golden/make_goldens_gman.py

Cases: tests/gman_seq.CASES.  For each, every output, cost, gradient (X per step, the learned SE, every parameter) and BatchNorm buffer
after the steps (tests/gman_seq.run) as a float64 fingerprint, stacked into one (keys, 5) tensor with its key list; the costs (float32
roundings of the float64 values, 2^-24 relative, far below the tests' 2^-20 floor) and the `num_batches_tracked` counters also as
values.  That keeps the fixture small.  The parameters come from each case's seed (gman_seq.seeded_state).  The reference runs under
gman_seq.cpu_batchnorm_fix: torch's CPU BatchNorm2d backward returns wrong input gradients for the permuted layouts the reference's
Conv2D produces at one node or B = T = 1."""
import gzip
import io
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
from gman_seq import CASES, FIXTURE, cpu_batchnorm_fix, fingerprint, model_for, reference_module, run  # noqa: E402

OUT = os.path.join(HERE, FIXTURE)
D = torch.float64


def _case(name):
    c = dict(CASES[name])
    with cpu_batchnorm_fix():
        got = run(model_for(c, reference_module().GMAN, "cpu", D), c, "cpu", D)
    c.update(values={k: (v if v.dtype == torch.int64 else v.float()) for k, v in got.items()
                     if k.startswith("cost.") or v.dtype == torch.int64},
             fingerprint_keys=list(got), fingerprints=torch.stack([fingerprint(v) for v in got.values()]))
    return c


def main():
    torch.set_default_dtype(D)         # the reference builds its one-hot in the default dtype
    cases = {name: _case(name) for name in CASES}
    for k, c in cases.items():
        print(f"{k}: cost {float(c['values']['cost.0']):.6f}")
    buf = io.BytesIO()
    torch.save(dict(cases=cases), buf)
    with gzip.GzipFile(OUT, "wb", compresslevel=9, mtime=0) as f:
        f.write(buf.getvalue())
    print(f"{os.path.basename(OUT)}  {os.path.getsize(OUT) / 1024:.0f} KB")


if __name__ == "__main__":
    main()
