"""Golden values for TGCN, TGCN2, A3TGCN and A3TGCN2 at 64 hidden channels, from the UNMODIFIED reference modules (imported through
oracle/refload.py on top of oracle/stubs), computed in float64.  Run in the build container only:   python tests/golden/make_goldens_tgcn64.py

The cases, their inputs and their loops are tests/tgcn64_seq.py's (CASES, data, run); each case's parameters come from its seed.  The fixture
holds, per case, the reference's loss and the fingerprints (tests/lstm64_seq.fingerprint) of its outputs and of every gradient.
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
from lstm64_seq import fingerprint  # noqa: E402
from tgcn64_seq import CASES, FIXTURE, SeqModel, data, run, seeded_state  # noqa: E402


def main():
    tg, at = refload.load("nn.recurrent.temporalgcn"), refload.load("nn.recurrent.attentiontemporalgcn")
    mods = {"TGCN": tg.TGCN, "TGCN2": tg.TGCN2, "A3TGCN": at.A3TGCN, "A3TGCN2": at.A3TGCN2}
    torch.set_default_dtype(torch.float64)
    out = {}
    for name, c in CASES.items():
        m = SeqModel(c, mods)
        m.load_state_dict({k: v.double() for k, v in seeded_state(c).items()})
        d = {k: v.double() if v.is_floating_point() else v for k, v in data(c).items()}
        res = run(m, c, d)
        fp = {"out": fingerprint(res["out"]), **{f"grad/{k}": fingerprint(g) for k, g in res.get("grads", {}).items()}}
        if "gH0" in res:
            fp["gH0"] = fingerprint(res["gH0"])
        out[name] = {"loss": None if res["loss"] is None else float(res["loss"].detach()), "fingerprints": fp}
        print(name, out[name]["loss"], len(fp))
    buf = io.BytesIO()
    torch.save(out, buf)
    with gzip.open(os.path.join(HERE, FIXTURE), "wb") as f:
        f.write(buf.getvalue())
    print(f"{FIXTURE}  {os.path.getsize(os.path.join(HERE, FIXTURE)) / 1024:.0f} KB")


if __name__ == "__main__":
    main()
