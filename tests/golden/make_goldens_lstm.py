"""Golden vectors for GConvLSTM and GCLSTM training at 32 hidden channels from the UNMODIFIED reference modules (imported through
oracle/refload.py on top of oracle/stubs, as make_goldens_gconvgru.py does).  Run in the build container only:
    python tests/golden/make_goldens_lstm.py

The loop is tests/lstm_seq.py's `run`, written in the test tree (not copied from the examples).  One gzip-compressed file, lstm_rows.pt.gz,
holds for both modules:
* chickenpox_K1_sym, chickenpox_K2_sym, chickenpox_K2_rw  -- examples/recurrent/gconvlstm_example.py's / gclstm_example.py's epoch:
                                                          (4, 32, K) over the 103 snapshots of the 20 % chickenpox train split, H and C
                                                          carried from None, cumulative MSE / 103; `rw` with lambda_max = 1.8
* metr_la_K2                                           -- (2, 32, 2) on the 207-node METR-LA-shaped graph, 12 steps carried from leaf
                                                          H0 / C0 (tests/lstm_seq.carried_state), dL/dH0 and dL/dC0 stored
* wikimaths_K2                                         -- (14, 32, 2) on the 1068-node WikiMaths graph over its first 3 snapshots, H and
                                                          C carried from None; the graph and series come from gconvgru_wikimaths.pt.gz
Every case stores every prediction, the cost and the gradient of every parameter; biases are set to non-zero values.  The K = 2 sym and rw
chickenpox cases share one parameter set."""
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
import lstm_seq  # noqa: E402

REF = {"gconvlstm": ("nn.recurrent.gconv_lstm", "GConvLSTM"), "gclstm": ("nn.recurrent.gc_lstm", "GCLSTM")}
CASES = [("chickenpox_K1_sym", "chickenpox", 4, 1, "sym", None), ("chickenpox_K2_sym", "chickenpox", 4, 2, "sym", None),
         ("chickenpox_K2_rw", "chickenpox", 4, 2, "rw", 1.8), ("metr_la_K2", "metr_la", 2, 2, "sym", None),
         ("wikimaths_K2", "wikimaths", 14, 2, "sym", None)]


def main():
    states, cases = {}, {}
    for module, (path, cls_name) in REF.items():
        cls = getattr(refload.load(path), cls_name)
        for name, data, F, K, norm, lam in CASES:
            skey = f"{module}_{data}_K{K}"
            seed = 40 + 10 * list(REF).index(module) + K + (0 if data == "chickenpox" else 3 if data == "metr_la" else 6)
            torch.manual_seed(seed)
            m = lstm_seq.RecurrentGCN(cls, F, K, norm)
            g = torch.Generator().manual_seed(seed + 1)
            with torch.no_grad():
                for n_, p in m.named_parameters():
                    if n_.endswith("bias") or n_.split(".")[-1].startswith("b_"):
                        p.copy_(torch.randn(p.shape, generator=g) * 0.1)
            if skey in states:
                m.load_state_dict(states[skey])
            else:
                states[skey] = {k: v.detach().clone() for k, v in m.state_dict().items()}
            lam_t = None if lam is None else torch.tensor(lam)
            outs, cost, H0, C0 = lstm_seq.run_case_data(m, data, HERE, lam_t)
            cost.backward()
            c = dict(module=module, data=data, F=F, K=K, normalization=norm, lambda_max=lam_t, state=skey,
                     out=outs.detach().clone(), loss=cost.detach().clone(),
                     grads={k: p.grad.detach().clone() for k, p in m.named_parameters()})
            if H0 is not None:
                c.update(gH0=H0.grad.clone(), gC0=C0.grad.clone())
            cases[f"{module}_{name}"] = c
            print(f"{module}_{name}: loss {float(cost):.6f}")
    buf = io.BytesIO()
    torch.save(dict(states=states, cases=cases), buf)
    out = os.path.join(HERE, lstm_seq.FIXTURE)
    with gzip.GzipFile(out, "wb", mtime=0) as f:
        f.write(buf.getvalue())
    print(f"{lstm_seq.FIXTURE}  {os.path.getsize(out) / 1024:.0f} KB")


if __name__ == "__main__":
    main()
