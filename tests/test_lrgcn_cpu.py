"""LRGCN without a GPU: the float64 RGCNConv oracle against a dense per-relation mean and the reference's stored results, the module's
parameter layout and seeded init against the reference's, the edge_type mapping, the packed-weight layout with its inverse gradient
mapping, and the routing predicate."""
import os

import pytest
import torch

from lrgcn_seq import (RGCNConv, check_reference, edge_types, load, oracle_run, rgcn, seeded_state, states_for)
from gconvgru_seq import chickenpox_train_split
from oracle import refload
from pytorch_geometric_temporal_b200 import ops
from pytorch_geometric_temporal_b200.nn.recurrent import LRGCN
from pytorch_geometric_temporal_b200.nn.recurrent.lrgcn import relation_ids
from wikimaths_seq import load as load_wikimaths

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
D = torch.float64


def test_oracle_against_dense_relation_means():
    g = torch.Generator().manual_seed(3)
    n, R = 9, 3
    ei = torch.tensor([[0, 1, 2, 2, 3, 4, 4, 5, 8, 0, 7, 7], [1, 1, 0, 0, 5, 4, 2, 3, 2, 6, 6, 6]])   # self loops, duplicates, isolated 8
    et = torch.tensor([0, 1, 0, 0, 2, 0, 1, 2, 0, 5, 1, 1])                                          # type 5 matches nothing
    x = torch.randn(n, 4, generator=g, dtype=D)
    p = dict(weight=torch.randn(R, 4, 3, generator=g, dtype=D), root=torch.randn(4, 3, generator=g, dtype=D),
             bias=torch.randn(3, generator=g, dtype=D))
    want = x @ p["root"] + p["bias"]
    for r in range(R):
        A = torch.zeros(n, n, dtype=D)
        for k in range(ei.size(1)):
            if et[k] == r:
                A[ei[1, k], ei[0, k]] += 1
        A = A / A.sum(1, keepdim=True).clamp(min=1)
        want = want + A @ x @ p["weight"][r]
    torch.testing.assert_close(rgcn(p, x, ei, et, R), want, rtol=1e-13, atol=1e-13)
    comp = torch.randn(R, 2, generator=g, dtype=D)
    V = torch.randn(2, 4, 3, generator=g, dtype=D)
    Wb = torch.einsum("rb,bio->rio", comp, V)
    torch.testing.assert_close(rgcn(dict(p, weight=V, comp=comp), x, ei, et, R), rgcn(dict(p, weight=Wb), x, ei, et, R))


def _graph(c):
    if c["graph"] == "chickenpox":
        return chickenpox_train_split()
    w = load_wikimaths(GOLDEN)
    return w["edge_index"], w["edge_weight"], w["X"], w["Y"]


@pytest.mark.parametrize("name", sorted(load(GOLDEN)["cases"]))
def test_oracle_matches_reference(name):
    c = load(GOLDEN)["cases"][name]
    ei, ew, X, Y = _graph(c)
    H0, C0 = states_for(c, X.shape[1], dtype=D)
    et = edge_types(c["types"], ei, ew.double() if c["types"] == "attr" else ew)
    outs, cost, leaves = oracle_run(c, X, Y, ei, et, H0, C0)
    cost.backward()
    check_reference(c, outs.detach(), cost, {k: v.grad for k, v in leaves.items()},
                    None if H0 is None else H0.grad, None if C0 is None else C0.grad)
    if name == "tutorial":                     # float ones as edge_type: relation 0 selects no edge
        assert all(float(v.grad.abs().max()) == 0 for k, v in leaves.items() if k.endswith((".weight", ".comp")) and "conv" in k)


@pytest.mark.parametrize("R,B", [(1, 1), (2, 2), (3, None), (2, None)])
def test_state_dict_and_seeded_init_match_reference(R, B):
    ours = LRGCN(5, 32, R, B)
    keys = [f"conv_{s}_{g}.{p}" for g in "ifco" for s in "xh" for p in ("weight", "comp", "root", "bias") if B is not None or p != "comp"]
    assert list(ours.state_dict()) == keys
    assert ours.conv_x_i.weight.shape == ((B or R), 5, 32) and ours.conv_h_o.root.shape == (32, 32)
    if not refload.available():
        pytest.skip("reference tree not present")
    import sys
    sys.path.insert(0, refload._STUBS)
    import torch_geometric.nn as tgnn
    tgnn.RGCNConv = RGCNConv
    ref_cls = refload.load("nn.recurrent.lrgcn").LRGCN
    torch.manual_seed(7)
    ref = ref_cls(5, 32, R, B)
    torch.manual_seed(7)
    ours = LRGCN(5, 32, R, B)
    assert list(ref.state_dict()) == list(ours.state_dict())
    for k, v in ref.state_dict().items():
        assert torch.equal(v, ours.state_dict()[k]), k


def test_relation_ids():
    nan, inf = float("nan"), float("inf")
    f = torch.tensor([0.0, 1.0, 1.5, -1.0, 2.0, nan, inf, -0.0, 1e30, 0.999999])
    assert relation_ids(f, 2).tolist() == [0, 1, -1, -1, -1, -1, -1, 0, -1, -1]
    assert relation_ids(f.half(), 3).tolist()[:5] == [0, 1, -1, -1, 2]
    i = torch.tensor([0, 1, 2, -1, 5, 1 << 40])
    assert relation_ids(i, 2).tolist() == [0, 1, -1, -1, -1, -1]
    assert relation_ids(i[:5].int(), 3).tolist() == [0, 1, 2, -1, -1]
    assert relation_ids(torch.ones(4), 1).tolist() == [-1] * 4           # the tutorial: float ones select no relation
    assert relation_ids(torch.tensor([True, False]), 2).tolist() == [1, 0]
    assert relation_ids(torch.empty(0), 2).numel() == 0


@pytest.mark.parametrize("R,B,cin,co", [(1, 1, 4, 32), (2, 2, 14, 32), (2, None, 5, 32), (1, None, 16, 64)])
def test_pack_layout_and_gradient_blocks(R, B, cin, co):
    """The packed layout of _rows_packed, emulated in float64, and _rows_spec as its inverse: every parameter block is where the pack puts
    it, so the kernel's dw / db blocks are the parameters' gradients (through autograd for the composed relation weights)."""
    torch.manual_seed(0)
    m = LRGCN(cin, co, R, B).double()
    with torch.no_grad():
        for c in m._convs():
            c.bias.normal_()
    C = cin + co
    w = torch.zeros(4 * co, (R + 1) * C, dtype=D)
    b = torch.zeros(4 * co, dtype=D)
    for gi, g in enumerate("ifco"):
        for s, off in (("x", 0), ("h", cin)):
            c = getattr(m, f"conv_{s}_{g}")
            blocks = torch.cat([c.root.unsqueeze(0), c.relation_weights()]).transpose(1, 2)
            for k in range(R + 1):
                w[gi * co:(gi + 1) * co, k * C + off:k * C + off + blocks.size(2)] = blocks[k]
            b[gi * co:(gi + 1) * co] += c.bias
    assert int(torch.count_nonzero(w)) == w.numel()                       # every column of the basis is some parameter's
    spec, params = m._rows_spec()
    dw = torch.randn_like(w)
    db = torch.randn(7 * co, dtype=D)
    grads = ops._spec_grads(spec, dw, db)
    for s, p, gr in zip(spec, params, grads):
        if s[0] == "wt":
            assert torch.equal(w[s[1]:s[1] + s[2], s[3]:s[3] + s[4]].t(), p.detach())
        else:
            assert s[1] % co == 0 and s[2] == co and p.shape == (co,)        # a gate's bias row block: b sums bias_x and bias_h
        assert gr.shape == p.shape
    torch.autograd.backward([p for p in params if p.requires_grad], [g for p, g in zip(params, grads) if p.requires_grad])
    for gi, g in enumerate("ifco"):                       # the composed weights' gradients, as in RGCNConv: dV = comp^T dW, dcomp = <dW_r, V_b>
        for s, off, width in (("x", 0, cin), ("h", cin, co)):
            c = getattr(m, f"conv_{s}_{g}")
            dW = torch.stack([dw[gi * co:(gi + 1) * co, (1 + r) * C + off:(1 + r) * C + off + width].t() for r in range(R)])
            torch.testing.assert_close(c.root.grad, dw[gi * co:(gi + 1) * co, off:off + width].t())
            if B is None:
                torch.testing.assert_close(c.weight.grad, dW)
            else:
                torch.testing.assert_close(c.weight.grad, torch.einsum("rb,rio->bio", c.comp.detach(), dW))
                torch.testing.assert_close(c.comp.grad, torch.einsum("rio,bio->rb", dW, c.weight.detach()))


class _Plan:
    num_nodes = 20


@pytest.mark.parametrize("cin,co,R,shape,dtype,training,fused,want", [
    (4, 32, 1, None, torch.float32, False, True, True), (16, 32, 2, None, torch.float32, True, True, True),
    (16, 64, 1, None, torch.float32, True, True, True), (4, 64, 2, None, torch.float32, False, True, False),
    (17, 32, 1, None, torch.float32, False, True, False), (4, 48, 1, None, torch.float32, False, True, False),
    (4, 32, 3, None, torch.float32, False, True, False), (4, 32, 2, (20, 31), torch.float32, False, True, False),
    (4, 32, 2, (20, 32), torch.float64, False, True, False), (4, 32, 2, (20, 32), torch.float32, True, False, False),
    (4, 32, 2, (20, 32), torch.float32, False, False, True)])
def test_routing_predicate(monkeypatch, cin, co, R, shape, dtype, training, fused, want):
    monkeypatch.setattr(ops, "lstm_rows_supported", lambda plan, variant, n_ops, c, o: n_ops <= 2 and c <= 16 and o in (32, 64))
    m = LRGCN(cin, co, R, 1)
    m.fused_training = fused
    X = torch.zeros(20, cin)
    H = None if shape is None else torch.zeros(shape, dtype=dtype)
    plans = [_Plan()] * ((R + 1) // 2)
    assert m._rows_ok(plans, X, H, None, training) is want
    assert m._rows_ok(plans, X.unsqueeze(0), None, None, training) is False
