"""The GMAN cases, shared by tests/golden/make_goldens_gman.py, the CPU and GPU GMAN tests and tests/perf/bench_gman.py.

Every case builds GMAN(L, K, d, num_his, bn_decay, steps_per_day, use_bias, mask) with parameters drawn from its seed, a learned SE and
runs `steps` training calls (train mode: batch statistics and running-statistic updates), each followed by the backward of a fixed random
projection of the output (gradients accumulate over the steps), then with `eval_call` one eval-mode call:
* unit_l1, unit_l2_mask   the reference's test_gman shapes: N = 50, num_his 12, num_pred 10, B = 32, K = d = 8; L = 1 with bias and
                          without mask, and L = 2 without bias and with mask
* k4_d16, k16_d4          16 heads of width 4 and 4 heads of width 16 (the logits scaled by 1/sqrt(d), the number of heads)
* steps_mask              two training steps then an eval call, with mask, bn_decay = 0.1
* steps_cumulative        the same with bn_decay = None (a cumulative running average), without mask
* pems                    the PEMS-BAY shape: N = 325, num_his = num_pred = 12, B = 2, L = 1, K = d = 8
The parameters, SE and the inputs come from the case's seed as float32 values, so a float64 run and a float32 run see the same numbers."""
import contextlib
import gzip
import io
import math
import os

import torch

from lstm64_seq import fingerprint  # noqa: F401  (re-exported for the tests)

FIXTURE = "gman.pt.gz"

_UNIT = dict(N=50, his=12, pred=10, B=32, K=8, d=8, bn_decay=0.1, spd=288)
CASES = {
    "unit_l1": dict(_UNIT, L=1, use_bias=True, mask=False, steps=1, eval_call=False, seed=601),
    "unit_l2_mask": dict(_UNIT, L=2, use_bias=False, mask=True, steps=1, eval_call=False, seed=602),
    "k4_d16": dict(N=20, his=6, pred=4, B=4, K=4, d=16, bn_decay=0.1, spd=24, L=1, use_bias=True, mask=False, steps=1,
                   eval_call=True, seed=603),
    "k16_d4": dict(N=20, his=6, pred=4, B=4, K=16, d=4, bn_decay=0.1, spd=24, L=1, use_bias=True, mask=False, steps=1,
                   eval_call=True, seed=604),
    "steps_mask": dict(N=30, his=8, pred=6, B=4, K=4, d=4, bn_decay=0.1, spd=48, L=1, use_bias=True, mask=True, steps=2,
                       eval_call=True, seed=605),
    "steps_cumulative": dict(N=30, his=8, pred=6, B=4, K=4, d=4, bn_decay=None, spd=48, L=1, use_bias=True, mask=False, steps=2,
                             eval_call=True, seed=606),
    "pems": dict(N=325, his=12, pred=12, B=2, K=8, d=8, bn_decay=0.1, spd=288, L=1, use_bias=True, mask=False, steps=1,
                 eval_call=False, seed=607),
}


def build(cls, c):
    return cls(c["L"], c["K"], c["d"], c["his"], c["bn_decay"], c["spd"], c["use_bias"], c["mask"])


def seeded_state(c, cls):
    """The parameters of case c from its seed (float32 values): conv weights N(0, 2 / (in + out)), BatchNorm weights 1 + N(0, 0.3),
    every other parameter N(0, 0.3), in sorted key order; the buffers keep their initial values."""
    m = build(cls, c)
    g = torch.Generator().manual_seed(c["seed"])
    names = dict(m.named_parameters())
    state = dict(m.state_dict())
    for k in sorted(names):
        shape = state[k].shape
        v = torch.randn(shape, generator=g, dtype=torch.float64)
        if k.endswith("_conv2d.weight"):
            v = v * math.sqrt(2.0 / (shape[0] + shape[1]))
        elif k.endswith("_batch_norm.weight"):
            v = 1 + 0.3 * v
        else:
            v = 0.3 * v
        state[k] = v.float()
    return state


def inputs(c, step):
    """(X (B, his, N), TE (B, his + pred, 2), G (B, pred, N)) of step `step` of case c, float32: X uniform in [0, 1), TE integer days
    and times of day from below zero to past a week and a day, plus a fraction in [0, 0.9) (truncated by the model), G N(0, 1)."""
    g = torch.Generator().manual_seed(c["seed"] * 10 + step)
    B, T = c["B"], c["his"] + c["pred"]
    X = torch.rand(B, c["his"], c["N"], generator=g)
    day = torch.randint(-9, 16, (B, T, 1), generator=g)
    tod = torch.randint(-c["spd"], 2 * c["spd"], (B, T, 1), generator=g)
    frac = torch.rand(B, T, 2, generator=g) * 0.9
    TE = torch.cat((day, tod), dim=-1).float() + torch.where(torch.cat((day, tod), -1) < 0, -frac, frac)
    G = torch.randn(B, c["pred"], c["N"], generator=g)
    return X, TE, G


def spatial_embedding(c):
    g = torch.Generator().manual_seed(c["seed"] + 1000)
    return torch.randn(c["N"], c["K"] * c["d"], generator=g)


def model_for(c, cls, device, dtype):
    m = build(cls, c)
    m.load_state_dict(seeded_state(c, cls))
    return m.to(device=device, dtype=dtype)


def run(m, c, device, dtype):
    """The case's training steps and eval call on model m.  -> {name: tensor}: out.<step>, out.eval, grad.X.<step>, grad.SE, grad.<param>
    and every BatchNorm buffer after the steps (buf.<key>), and the costs (cost.<step>)."""
    SE = spatial_embedding(c).to(device=device, dtype=dtype).requires_grad_(True)
    got = {}
    m.train()
    for s in range(c["steps"]):
        X, TE, G = inputs(c, s)
        X = X.to(device=device, dtype=dtype).requires_grad_(True)
        out = m(X, SE, TE.to(device=device, dtype=dtype))
        cost = (out * G.to(device=device, dtype=dtype)).sum()
        cost.backward()
        got[f"out.{s}"], got[f"cost.{s}"], got[f"grad.X.{s}"] = out.detach(), cost.detach().view(1), X.grad
    got["grad.SE"] = SE.grad
    for k, p in m.named_parameters():
        got[f"grad.{k}"] = p.grad if p.grad is not None else torch.zeros_like(p)
    for k, b in m.state_dict().items():
        if "running" in k or "num_batches" in k:
            got[f"buf.{k}"] = b.detach().clone()
    if c["eval_call"]:
        m.eval()
        X, TE, _ = inputs(c, 99)
        with torch.no_grad():
            got["out.eval"] = m(X.to(device=device, dtype=dtype), SE.detach(), TE.to(device=device, dtype=dtype))
        m.train()
    return got


class _ContiguousGrad(torch.autograd.Function):
    """Identity whose backward hands on a contiguous gradient."""

    @staticmethod
    def forward(ctx, x):
        return x.view_as(x)

    @staticmethod
    def backward(ctx, g):
        return g.contiguous()


@contextlib.contextmanager
def cpu_batchnorm_fix():
    """torch's CPU BatchNorm2d backward (2.11) mis-reads the permuted gradient the reference's Conv2D hands it when the (B, C, N, T)
    activation is also a channels-last tensor (one node, or B = T = 1: the spatial embedding's (1, D, N, 1)), and returns a wrong
    input gradient (checked against finite differences).  Inside this block every BatchNorm2d receives a contiguous gradient, which
    changes no value of the computation; the forward is untouched."""
    orig = torch.nn.BatchNorm2d.forward
    torch.nn.BatchNorm2d.forward = lambda self, x: _ContiguousGrad.apply(orig(self, x))
    try:
        yield
    finally:
        torch.nn.BatchNorm2d.forward = orig


def reference_module():
    """The unmodified reference nn/attention/gman.py."""
    from oracle import refload
    return refload.load("nn.attention.gman")


def load(golden_dir):
    """The goldens (tests/golden/make_goldens_gman.py), each case's stacked fingerprints unpacked into {key: fingerprint}."""
    with gzip.open(os.path.join(golden_dir, FIXTURE), "rb") as f:
        g = torch.load(io.BytesIO(f.read()), weights_only=False)
    for c in g["cases"].values():
        c["fingerprints"] = dict(zip(c.pop("fingerprint_keys"), c["fingerprints"]))
    return g
