"""Autograd-aware wrappers over the C ABI (stmp_spmm, fused DCRNN sequence, gate epilogues)."""
import ctypes
from typing import Optional

import torch

from . import _lib
from .plan import GraphPlan, _require_cuda


def _f32c(t: torch.Tensor, name: str) -> torch.Tensor:
    _require_cuda(t, name)
    if t.dtype != torch.float32:
        raise RuntimeError(f"{name} must be float32, got {t.dtype}")
    return t.contiguous()


def _require_numel(fn: str, n: int, **operands):
    """Raises unless every operand given (None: absent) holds exactly `n` elements, the count its kernel indexes: the elementwise and
    epilogue kernels take one row count for all their operands and trust it."""
    for name, t in operands.items():
        if t is not None and t.numel() != n:
            raise RuntimeError(f"{fn}: {name} has {t.numel()} elements, the kernel indexes {n}")


def spmm_raw(plan: GraphPlan, op: int, x: torch.Tensor, transposed: bool = False, alpha: float = 1.0,
             z: Optional[torch.Tensor] = None, beta: float = 0.0, att: Optional[torch.Tensor] = None,
             out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """y = alpha * A_op x + beta * z on (N,F) or (B,N,F) tensors; no autograd."""
    x = _f32c(x, "x")
    squeeze = x.dim() == 2
    x3 = x.unsqueeze(0) if squeeze else x
    if x3.dim() != 3 or x3.size(1) != plan.num_nodes:
        raise RuntimeError(f"expected (..., {plan.num_nodes}, F) features, got {tuple(x.shape)}")
    B, N, F = x3.shape
    y = torch.empty_like(x3) if out is None else out
    z3 = None
    if z is not None:
        z3 = _f32c(z, "z")
        z3 = z3.unsqueeze(0) if z3.dim() == 2 else z3
        if z3.shape != x3.shape:                       # the kernel reads z with x's batch and row strides
            raise RuntimeError(f"z must have the shape of x {tuple(x.shape)}, got {tuple(z.shape)}")
    a3 = None
    if att is not None:
        a3 = _f32c(att, "att")
        if a3.shape != (B, N, N):
            raise RuntimeError(f"attention must be ({B},{N},{N}), got {tuple(a3.shape)}")
    with torch.cuda.device(x.device):
        rc = _lib.lib().stmp_spmm(plan.handle, op, int(transposed), B, F, _lib.ptr(x3), F, N * F, _lib.ptr(y), F, N * F,
                                  alpha, _lib.ptr(z3), F, N * F, beta, _lib.ptr(a3), _lib.stream_ptr())
    _lib.check(rc)
    return y.squeeze(0) if squeeze else y


class _SpMM(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, z, att, plan, op, alpha, beta):
        ctx.plan, ctx.op, ctx.alpha, ctx.beta = plan, op, alpha, beta
        ctx.has_z, ctx.has_att = z is not None, att is not None
        ctx.save_for_backward(x if att is not None else None, att)
        return spmm_raw(plan, op, x, False, alpha, z, beta, att)

    @staticmethod
    def backward(ctx, gy):
        x, att = ctx.saved_tensors
        gy = gy.contiguous()
        gx = gz = gatt = None
        if ctx.needs_input_grad[0]:
            gx = spmm_raw(ctx.plan, ctx.op, gy, True, ctx.alpha, None, 0.0, att)
        if ctx.has_z and ctx.needs_input_grad[1]:
            gz = gy * ctx.beta
        if ctx.has_att and ctx.needs_input_grad[2]:
            # (N, F) features carry a (1, N, N) attention; the kernel writes gatt row-major whatever att's strides are
            gy3, x3 = (gy.unsqueeze(0), x.unsqueeze(0)) if gy.dim() == 2 else (gy, x)
            B, N, F = gy3.shape
            gatt = torch.zeros(att.shape, dtype=att.dtype, device=att.device)
            with torch.cuda.device(gy.device):
                rc = _lib.lib().stmp_spmm_att_grad(ctx.plan.handle, ctx.op, B, F, _lib.ptr(gy3), F, N * F,
                                                   _lib.ptr(x3.contiguous()), F, N * F, _lib.ptr(gatt), _lib.stream_ptr())
            _lib.check(rc)
            if ctx.alpha != 1.0:
                gatt = gatt * ctx.alpha
        return gx, gz, gatt, None, None, None, None


def spmm(plan: GraphPlan, op: int, x: torch.Tensor, alpha: float = 1.0, z: Optional[torch.Tensor] = None,
         beta: float = 0.0, att: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Differentiable y = alpha * A_op x + beta * z (gather -> weighted scatter-add, K1/K3)."""
    return _SpMM.apply(x, z, att, plan, op, float(alpha), float(beta))


_SEQ_WS = {}
_WGRAD_WS = {}


def _seq_workspace(plan: GraphPlan, T: int, cin: int, device) -> torch.Tensor:
    """Per-(device, stream) workspace of the fused sequence kernels (stmp_seq_workspace_bytes), grown on demand and reused: launches on
    one stream are ordered, so consecutive calls may share it."""
    need = int(_lib.lib().stmp_seq_workspace_bytes(plan.handle, T, cin))
    key = (torch.device(device).index, torch.cuda.current_stream(device).cuda_stream)
    buf = _SEQ_WS.get(key)
    if buf is None or buf.numel() < need:
        buf = torch.empty(max(need, 1), dtype=torch.uint8, device=device)
        _SEQ_WS[key] = buf
    return buf


def _wgrad_workspace(device, bytes_entry, *shape) -> torch.Tensor:
    """Per-(device, stream, entry, shape) workspace of a weight-gradient entry, `bytes_entry(*shape)` bytes (its *_wgrad_workspace_bytes,
    asked on the first call only) and then reused as it is: launches on one stream are ordered, so consecutive calls may share it."""
    key = (device, torch.cuda.current_stream(device).cuda_stream, bytes_entry.__name__, *shape)
    buf = _WGRAD_WS.get(key)
    if buf is None:
        buf = _WGRAD_WS[key] = torch.empty(int(bytes_entry(*shape)), device=device, dtype=torch.uint8)
    return buf


def dcrnn_seq_supported(plan: GraphPlan, cin: int, cout: int, K: int) -> bool:
    return bool(_lib.lib().stmp_dcrnn_seq_supported(plan.handle, cin, cout, K))


def dcrnn_seq_fwd(plan: GraphPlan, x: torch.Tensor, wz, wr, wh, bz, br, bh, K: int, h0=None,
                  win_start: Optional[torch.Tensor] = None, horizon: Optional[int] = None, stash: bool = False,
                  wimage: Optional[torch.Tensor] = None):
    """Fused DCRNN recurrence.  x: (B,T,N,Cin) windows, or -- with win_start (int64 [B]) and horizon --
    the resident series (T_total,N,Cin) from which window b = series[win_start[b]:win_start[b]+horizon]
    is read in-kernel (index-batching).  Returns out (B,T,N,Cout) [, stash (B,T,3,N,Cout)]."""
    x = _f32c(x, "X")
    N = plan.num_nodes
    cout = wz.size(-1)
    if win_start is None:
        if x.dim() != 4 or x.size(2) != N:
            raise RuntimeError(f"X must be (B,T,{N},Cin), got {tuple(x.shape)}")
        B, T, _, cin = x.shape
        bstride, tstride = T * N * cin, N * cin
        ws = None
    else:
        if x.dim() != 3 or x.size(1) != N:
            raise RuntimeError(f"series must be (T_total,{N},Cin), got {tuple(x.shape)}")
        _require_cuda(win_start, "win_start")
        ws = win_start.to(torch.int64).contiguous()
        B, T, cin = ws.numel(), int(horizon), x.size(2)
        bstride, tstride = 0, N * cin
    if wz.size(2) != cin + cout:
        raise RuntimeError(f"DConv weight expects {wz.size(2)} input channels, got Cin+Cout={cin + cout}")
    out = torch.empty((B, T, N, cout), dtype=torch.float32, device=x.device)
    st = torch.empty((B, T, 3, N, cout), dtype=torch.float32, device=x.device) if stash else None
    if B == 0 or T == 0:   # nothing to launch (empty tensors have NULL data pointers)
        return (out, st) if stash else out
    h0c = None if h0 is None else _f32c(h0, "H")
    _require_numel("dcrnn_seq_fwd", B * N * cout, h0=h0c)                # every window reads its own (N, cout) state
    args = [_f32c(w.detach(), "weight") for w in (wz, wr, wh)]
    bs = [None if b is None else _f32c(b.detach(), "bias") for b in (bz, br, bh)]
    with torch.cuda.device(x.device):
        rc = _lib.lib().stmp_dcrnn_seq_fwd(plan.handle, B, T, cin, cout, K, _lib.ptr(x), _lib.ptr(ws), bstride, tstride,
                                           _lib.ptr(args[0]), _lib.ptr(args[1]), _lib.ptr(args[2]), _lib.ptr(bs[0]),
                                           _lib.ptr(bs[1]), _lib.ptr(bs[2]), _lib.ptr(h0c), _lib.ptr(out), _lib.ptr(st),
                                           _lib.ptr(wimage), _lib.ptr(_seq_workspace(plan, T, cin, x.device)), _lib.stream_ptr())
    _lib.check(rc)
    return (out, st) if stash else out


def gru_seq_supported(plan: GraphPlan, n_ops: int, cin: int, cout: int) -> bool:
    return bool(_lib.lib().stmp_gru_seq_supported(plan.handle, n_ops, cin, cout))


def gru_seq_fwd(plan: GraphPlan, n_ops: int, x: torch.Tensor, wcat: torch.Tensor, bcat: torch.Tensor, h0=None,
                h0_shared: bool = False, wimage: Optional[torch.Tensor] = None, stash: bool = False):
    """Generic fused graph-GRU recurrence (stmp_gru_seq_fwd).  x (B,T,N,Cin) -> out (B,T,N,32) [, stash (B,T,3,N,32) = (Z, R, H~)
    per step, the operand of the backward].  h0: (B,N,32), or (N,32)/(1,N,32) with h0_shared=True (every window starts from the same
    state), or None."""
    x = _f32c(x, "X")
    N = plan.num_nodes
    if x.dim() != 4 or x.size(2) != N:
        raise RuntimeError(f"X must be (B,T,{N},Cin), got {tuple(x.shape)}")
    B, T, _, cin = x.shape
    wcat, bcat = _f32c(wcat, "wcat"), _f32c(bcat, "bcat")
    if wcat.shape != (96, 112) or bcat.numel() != 96:
        raise RuntimeError("wcat must be (96,112) and bcat (96,)")
    out = torch.empty((B, T, N, 32), dtype=torch.float32, device=x.device)
    st = torch.empty((B, T, 3, N, 32), dtype=torch.float32, device=x.device) if stash else None
    if B == 0 or T == 0:
        return (out, st) if stash else out
    h0c, hs = None, 0
    if h0 is not None:
        h0c = _f32c(h0, "H")
        hs = 0 if h0_shared else N * 32
        _require_numel("gru_seq_fwd", N * 32 if h0_shared else B * N * 32, h0=h0c)   # the kernel reads h0 at batch stride hs
    with torch.cuda.device(x.device):
        rc = _lib.lib().stmp_gru_seq_fwd(plan.handle, n_ops, B, T, cin, _lib.ptr(x), None, T * N * cin, N * cin, _lib.ptr(wcat),
                                         _lib.ptr(bcat), _lib.ptr(h0c), hs, _lib.ptr(out), _lib.ptr(st), _lib.ptr(wimage),
                                         _lib.ptr(_seq_workspace(plan, T, cin, x.device)), _lib.stream_ptr())
    _lib.check(rc)
    return (out, st) if stash else out


def gru_bwd_supported(plan: GraphPlan, n_ops: int, cin: int, cout: int) -> bool:
    return bool(_lib.lib().stmp_gru_bwd_supported(plan.handle, n_ops, cin, cout))


def gru_bwd_basis_ld(n_ops: int, cin: int) -> int:
    """Row pitch of the graph-GRU bases [U | Op0 U | ..]: (n_ops+1)(cin+32) rounded up to 8 floats."""
    return ((n_ops + 1) * (cin + 32) + 7) // 8 * 8


def gru_pack_bwd_weights(n_ops: int, cin: int, wcat: torch.Tensor):
    """(whsT (32, (n_ops+1)(cin+32)), wzrT (64, ..)): the backward GEMMs' weights in basis order from the forward's wcat, one launch."""
    nb = (n_ops + 1) * (cin + 32)
    whsT = torch.empty(32, nb, device=wcat.device, dtype=torch.float32)
    wzrT = torch.empty(64, nb, device=wcat.device, dtype=torch.float32)
    with torch.cuda.device(wcat.device):
        _lib.check(_lib.lib().stmp_gru_pack_bwd_weights(n_ops, cin, _lib.ptr(_f32c(wcat, "wcat")), _lib.ptr(whsT), _lib.ptr(wzrT),
                                                        _lib.stream_ptr()))
    return whsT, wzrT


def gru_bwd_basis(plan: GraphPlan, n_ops: int, x, out, h0, stash, S1, S2):
    """S1 / S2 (T*B, N, ld) <- bases of [X_t | H_{t-1}] and [X_t | H_{t-1}*R_t] for every (t, b): one launch."""
    B, T, N, Ci = x.shape
    with torch.cuda.device(x.device):
        _lib.check(_lib.lib().stmp_gru_bwd_basis(plan.handle, n_ops, B, T, Ci, _lib.ptr(x), T * N * Ci, N * Ci, _lib.ptr(out), _lib.ptr(h0),
                                                 N * 32, _lib.ptr(stash), _lib.ptr(S1), _lib.ptr(S2), S1.size(-1), _lib.stream_ptr()))


def gru_bwd_seq(plan: GraphPlan, n_ops: int, cin: int, gout, out, h0, stash, whsT, wzrT, dph_all, dpzr_all, dx, dh0):
    """The reverse-time recurrence of the graph-GRU backward in one persistent launch (one CTA or CTA pair per window)."""
    B, T, N, _ = gout.shape
    with torch.cuda.device(gout.device):
        _lib.check(_lib.lib().stmp_gru_bwd_seq(plan.handle, n_ops, B, T, cin, _lib.ptr(gout), _lib.ptr(out), _lib.ptr(h0), N * 32,
                                               _lib.ptr(stash), _lib.ptr(whsT), _lib.ptr(wzrT), _lib.ptr(dph_all), _lib.ptr(dpzr_all),
                                               _lib.ptr(dx), _lib.ptr(dh0), _lib.stream_ptr()))


def gru_bwd_wgrad(n_ops: int, cin: int, S1, S2, dpzr_all, dph_all, has_bias: bool):
    """(dwcat (96, 112), dbcat (96,) or None): gradients of the forward's prepacked weights over all (t, b, n) rows, two launches."""
    dev = S1.device
    ws = _wgrad_workspace(dev, _lib.lib().stmp_gru_bwd_wgrad_workspace_bytes, n_ops, cin)
    dwcat = torch.empty(96, 112, device=dev, dtype=torch.float32)
    dbcat = torch.empty(96, device=dev, dtype=torch.float32) if has_bias else None
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().stmp_gru_bwd_wgrad(n_ops, cin, S1.size(0) * S1.size(1), S1.size(-1), _lib.ptr(S1), _lib.ptr(S2),
                                                 _lib.ptr(dpzr_all), _lib.ptr(dph_all), _lib.ptr(ws), _lib.ptr(dwcat), _lib.ptr(dbcat),
                                                 _lib.stream_ptr()))
    return dwcat, dbcat


def _spec_grads(spec, dw, db):
    """Parameter gradients as blocks of packed weight / bias gradients: ("w", row, n_rows, col, n_cols) -> dw[row:row+n_rows, col:col+n_cols]
    (("wt", ...) -> its transpose), ("b", row, n_rows) -> db[row:row+n_rows].  Parameters that share a block of db each get their own copy,
    so no two .grad tensors alias."""
    grads, dbs = [None] * len(spec), None
    for i, s in enumerate(spec):
        if s[0] in ("w", "wt"):
            grads[i] = dw[s[1]:s[1] + s[2], s[3]:s[3] + s[4]]
            if s[0] == "wt":
                grads[i] = grads[i].t()
        else:
            if dbs is None:
                dbs = db.expand(sum(1 for q in spec if q[0] == "b"), db.numel()).clone()
            grads[i] = dbs[sum(1 for q in spec[:i] if q[0] == "b"), s[1]:s[1] + s[2]]
    return grads


class _GruSeqFn(torch.autograd.Function):
    """Training form of the generic fused graph-GRU recurrence.  forward = `stmp_gru_seq_fwd` with a stash: the same launch as inference,
    so the output is bit-identical to the `no_grad` one.  backward = pack -> basis -> reverse-time recurrence -> weight gradients
    (`stmp_gru_pack_bwd_weights`, `stmp_gru_bwd_basis`, `stmp_gru_bwd_seq`, `stmp_gru_bwd_wgrad`): dX (when x requires grad), dH0 (when
    h0 requires grad), dwcat and dbcat.  `params` receive their gradients as blocks of dwcat / dbcat, described by `spec`:
    ("w", row, n_rows, col, n_cols) -> dwcat[row:row+n_rows, col:col+n_cols], ("b", row, n_rows) -> dbcat[row:row+n_rows] -- so a module
    whose prepacked weights are a cached fold of its parameters needs no differentiable fold."""

    @staticmethod
    def forward(ctx, plan, n_ops, x, h0, wcat, bcat, wimage, spec, *params):
        x = _f32c(x.detach(), "X")
        h0c = None if h0 is None else _f32c(h0.detach(), "H")
        out, stash = gru_seq_fwd(plan, n_ops, x, wcat, bcat, h0=h0c, wimage=wimage, stash=True)
        ctx.plan, ctx.n_ops, ctx.spec, ctx.has_h0 = plan, n_ops, spec, h0 is not None
        ctx.save_for_backward(x, h0c, out, stash, wcat)
        return out

    @staticmethod
    def backward(ctx, gout):
        x, h0, out, stash, wcat = ctx.saved_tensors
        plan, n_ops = ctx.plan, ctx.n_ops
        B, T, N, Ci = x.shape
        f32 = dict(device=x.device, dtype=torch.float32)
        gout = _f32c(gout, "gout")
        whsT, wzrT = gru_pack_bwd_weights(n_ops, Ci, wcat)
        ld = gru_bwd_basis_ld(n_ops, Ci)
        S1 = torch.empty(T * B, N, ld, **f32)
        S2 = torch.empty(T * B, N, ld, **f32)
        dph_all = torch.empty(T, B, N, 32, **f32)
        dpzr_all = torch.empty(T, B, N, 64, **f32)
        dX = torch.empty(x.shape, **f32) if ctx.needs_input_grad[2] else None
        dH0 = torch.empty(B, N, 32, **f32)
        gru_bwd_basis(plan, n_ops, x, out, h0, stash, S1, S2)
        gru_bwd_seq(plan, n_ops, Ci, gout, out, h0, stash, whsT, wzrT, dph_all, dpzr_all, dX, dH0)
        grads = [None] * len(ctx.spec)
        if any(ctx.needs_input_grad[8:]):
            dwcat, dbcat = gru_bwd_wgrad(n_ops, Ci, S1, S2, dpzr_all, dph_all, any(s[0] == "b" for s in ctx.spec))
            grads = _spec_grads(ctx.spec, dwcat, dbcat)
        gH0 = dH0 if (ctx.has_h0 and ctx.needs_input_grad[3]) else None
        return (None, None, dX, gH0, None, None, None, None, *grads)


def gru_seq_train(plan: GraphPlan, n_ops: int, x, h0, wcat, bcat, wimage, spec, params) -> torch.Tensor:
    """Differentiable (w.r.t. x, h0 and `params`, see _GruSeqFn) fused graph-GRU recurrence.  x (B,T,N,Cin), h0 (B,N,32) or None."""
    return _GruSeqFn.apply(plan, n_ops, x, h0, wcat, bcat, wimage, tuple(spec), *params)


def gru_rows_supported(plan: GraphPlan, n_ops: int, cin: int, cout: int) -> bool:
    return bool(_lib.lib().stmp_gru_rows_supported(plan.handle, n_ops, cin, cout))


def gru_rows_basis_ld(n_ops: int, cin: int, cout: int = 32) -> int:
    """Row pitch of the row-split cell's weight-gradient bases: (n_ops+1)(cin+cout) rounded up to 8 floats."""
    return ((n_ops + 1) * (cin + cout) + 7) // 8 * 8


def _gru_rows_entry(cout: int, what: str):
    """stmp_gru_rows_<what> at 32 hidden channels, stmp_gru_wide_rows_<what> at 64; the two families take the same arguments."""
    if cout not in (32, 64):
        raise RuntimeError(f"the row-split graph-GRU cell serves 32 or 64 hidden channels, not {cout}")
    return getattr(_lib.lib(), ("stmp_gru_wide_rows_" if cout == 64 else "stmp_gru_rows_") + what)


def gru_rows_pack_weights(n_ops: int, cin: int, wx, wh, bx=None, bh=None):
    """(w (3 cout, (n_ops+1)(cin+cout)), b (3 cout,)): the row-split cell's packed weights from the parameters' layout -- wx (3, n_ops+1, cout,
    cin), wh (3, n_ops+1, cout, cout), bx / bh (3, cout) or None, cout = 32 or 64 -- in one launch (stmp_gru_rows_pack_weights or
    stmp_gru_wide_rows_pack_weights)."""
    wx, wh = _f32c(wx, "wx"), _f32c(wh, "wh")
    cout = wh.size(-1) if wh.dim() == 4 else 32
    if wx.shape != (3, n_ops + 1, cout, cin) or wh.shape != (3, n_ops + 1, cout, cout):
        raise RuntimeError("gru_rows_pack_weights: wx must be (3, n_ops+1, cout, cin) and wh (3, n_ops+1, cout, cout)")
    bx = None if bx is None else _f32c(bx, "bx")
    bh = None if bh is None else _f32c(bh, "bh")
    w = torch.empty(3 * cout, (n_ops + 1) * (cin + cout), device=wx.device, dtype=torch.float32)
    b = torch.empty(3 * cout, device=wx.device, dtype=torch.float32)
    with torch.cuda.device(wx.device):
        _lib.check(_gru_rows_entry(cout, "pack_weights")(n_ops, cin, _lib.ptr(wx), _lib.ptr(wh), _lib.ptr(bx), _lib.ptr(bh), _lib.ptr(w),
                                                         _lib.ptr(b), _lib.stream_ptr()))
    return w, b


def gru_rows_fwd(plan: GraphPlan, n_ops: int, x: torch.Tensor, h: Optional[torch.Tensor], w: torch.Tensor, b: torch.Tensor,
                 train: bool = False):
    """Row-split graph-GRU cell (stmp_gru_rows_fwd, or stmp_gru_wide_rows_fwd for packed weights of 192 rows) on one graph: x (N, cin),
    h (N, cout) or None -> H' (N, cout), cout = w.size(0) / 3.  With `train`, returns (H', stash (3, N, cout), S1, S2) -- the operands of
    gru_rows_bwd / gru_rows_wgrad; S2 is S1 when h is None."""
    x, w, b = _f32c(x, "X"), _f32c(w, "w"), _f32c(b, "b")
    N, cin = x.shape
    cout = w.size(0) // 3
    f32 = dict(device=x.device, dtype=torch.float32)
    out = torch.empty(N, cout, **f32)
    hc = None if h is None else _f32c(h, "H")
    scr = torch.empty(N, 3 * cout, **f32) if hc is not None else None
    st = S1 = S2 = None
    ld = gru_rows_basis_ld(n_ops, cin, cout)
    if train:
        st = torch.empty(3, N, cout, **f32)
        S1 = torch.empty(N, ld, **f32)
        S2 = torch.empty(N, ld, **f32) if hc is not None else None
    with torch.cuda.device(x.device):
        _lib.check(_gru_rows_entry(cout, "fwd")(plan.handle, n_ops, cin, _lib.ptr(x), _lib.ptr(hc), _lib.ptr(w), _lib.ptr(b), _lib.ptr(scr),
                                                _lib.ptr(out), _lib.ptr(st), _lib.ptr(S1), _lib.ptr(S2), ld, _lib.stream_ptr()))
    if not train:
        return out
    return out, st, S1, S1 if S2 is None else S2


def gru_rows_bwd(plan: GraphPlan, n_ops: int, gout, h, stash, w, want_dx: bool, want_dh: bool, cin: int):
    """(dph (N, cout), dpzr (N, 2 cout), dx (N, cin) or None, dh (N, cout) or None) of the row-split cell (stmp_gru_rows_bwd, or
    stmp_gru_wide_rows_bwd when gout has 64 channels)."""
    gout = _f32c(gout, "gout")
    N, cout = gout.shape
    f32 = dict(device=gout.device, dtype=torch.float32)
    scr = torch.empty(int(_gru_rows_entry(cout, "scratch_bytes")(plan.handle)) // 4, **f32)
    dph, dpzr = torch.empty(N, cout, **f32), torch.empty(N, 2 * cout, **f32)
    dx = torch.empty(N, cin, **f32) if want_dx else None
    dh = torch.empty(N, cout, **f32) if want_dh else None
    with torch.cuda.device(gout.device):
        _lib.check(_gru_rows_entry(cout, "bwd")(plan.handle, n_ops, cin, _lib.ptr(gout), _lib.ptr(h), _lib.ptr(stash), _lib.ptr(w),
                                                _lib.ptr(scr), _lib.ptr(dph), _lib.ptr(dpzr), _lib.ptr(dx), _lib.ptr(dh), _lib.stream_ptr()))
    return dph, dpzr, dx, dh


def gru_rows_wgrad(n_ops: int, cin: int, S1, S2, dpzr, dph, has_bias: bool):
    """(dw (3 cout, (n_ops+1)(cin+cout)), db (3 cout,) or None): the packed weights' gradients of the row-split cell, two launches; cout =
    dph.size(1)."""
    dev = S1.device
    cout = dph.size(1)
    ws = _wgrad_workspace(dev, _gru_rows_entry(cout, "wgrad_workspace_bytes"), n_ops, cin)
    dw = torch.empty(3 * cout, (n_ops + 1) * (cin + cout), device=dev, dtype=torch.float32)
    db = torch.empty(3 * cout, device=dev, dtype=torch.float32) if has_bias else None
    with torch.cuda.device(dev):
        _lib.check(_gru_rows_entry(cout, "wgrad")(n_ops, cin, S1.size(0), S1.size(1), _lib.ptr(S1), _lib.ptr(S2), _lib.ptr(dpzr), _lib.ptr(dph),
                                                  _lib.ptr(ws), _lib.ptr(dw), _lib.ptr(db), _lib.stream_ptr()))
    return dw, db


class _GruRowsFn(torch.autograd.Function):
    """Training form of the row-split graph-GRU cell (32 or 64 hidden channels, from the packed weights), the twin of _GruSeqFn for graphs
    of any size.  forward = `stmp_gru_rows_fwd` (`stmp_gru_wide_rows_fwd`) with the
    stash and the weight-gradient bases (the inference launches, so the output is bit-identical to the `no_grad` one); backward =
    `stmp_gru_rows_bwd` + `stmp_gru_rows_wgrad`: dX (when x requires grad), dH (when h is given and requires grad) and the packed weights'
    gradients, handed to `params` as blocks described by `spec` (see _spec_grads)."""

    @staticmethod
    def forward(ctx, plan, n_ops, x, h, w, b, spec, *params):
        x = _f32c(x.detach(), "X")
        hc = None if h is None else _f32c(h.detach(), "H")
        out, stash, S1, S2 = gru_rows_fwd(plan, n_ops, x, hc, w, b, train=True)
        ctx.plan, ctx.n_ops, ctx.spec, ctx.cin = plan, n_ops, spec, x.size(1)
        ctx.save_for_backward(hc, stash, S1, S2, w)
        return out

    @staticmethod
    def backward(ctx, gout):
        h, stash, S1, S2, w = ctx.saved_tensors
        want_dh = h is not None and ctx.needs_input_grad[3]
        dph, dpzr, dx, dh = gru_rows_bwd(ctx.plan, ctx.n_ops, gout, h, stash, w, ctx.needs_input_grad[2], want_dh, ctx.cin)
        grads = [None] * len(ctx.spec)
        if any(ctx.needs_input_grad[7:]):
            dw, db = gru_rows_wgrad(ctx.n_ops, ctx.cin, S1, S2, dpzr, dph, any(s[0] == "b" for s in ctx.spec))
            grads = _spec_grads(ctx.spec, dw, db)
        return (None, None, dx, dh, None, None, None, *grads)


def gru_rows_train(plan: GraphPlan, n_ops: int, x, h, w, b, spec, params) -> torch.Tensor:
    """Differentiable (w.r.t. x, h and `params`, see _GruRowsFn) row-split graph-GRU cell.  x (N, cin), h (N, cout) or None (zeros, no dH)."""
    return _GruRowsFn.apply(plan, n_ops, x, h, w, b, tuple(spec), *params)


# GConvLSTM / GCLSTM at 64 hidden channels: from this many nodes on, inference with in_channels % 4 == 0 takes the SpMM + wgmma route
# (gemm_lstm).  Below it the 64-wide row-split cell's one launch is faster; above it, its 16-row tiles need a second wave of CTAs on an
# H100 (132 SMs, one CTA per SM) and the wgmma route is faster on the device (DESIGN §4o, tests/perf/bench_lstm64.py).
LSTM_WIDE_ROWS_GEMM_NODES = 2048


def lstm_rows_for_no_grad(plan: GraphPlan, cin: int, cout: int) -> bool:
    """Whether a `no_grad` call inside the row-split envelope takes the row-split LSTM cell: always at 32 channels; at 64 unless the SpMM
    + wgmma route serves it (cin % 4 == 0) on a graph of LSTM_WIDE_ROWS_GEMM_NODES nodes or more."""
    return cout != 64 or cin % 4 != 0 or plan.num_nodes < LSTM_WIDE_ROWS_GEMM_NODES


def lstm_rows_supported(plan: GraphPlan, variant: int, n_ops: int, cin: int, cout: int) -> bool:
    return bool(_lib.lib().stmp_lstm_rows_supported(plan.handle, variant, n_ops, cin, cout))


def lstm_rows_nb(variant: int, n_ops: int, cin: int, cout: int = 32) -> int:
    """Basis columns of the row-split LSTM cell: (n_ops+1)(cin+cout) for GConvLSTM ([X | H | Op X | Op H]), cin + cout(n_ops+1) for
    GCLSTM."""
    return cin + cout * (n_ops + 1) if variant == _lib.LSTM_GC else (n_ops + 1) * (cin + cout)


def lstm_rows_basis_ld(variant: int, n_ops: int, cin: int, cout: int = 32) -> int:
    """Row pitch of the row-split LSTM cell's weight-gradient basis: nb rounded up to 8 floats."""
    return (lstm_rows_nb(variant, n_ops, cin, cout) + 7) // 8 * 8


def _lstm_rows_entry(cout: int, what: str):
    """stmp_lstm_rows_<what> at 32 hidden channels, stmp_lstm_wide_rows_<what> at 64; the two families take the same arguments."""
    if cout not in (32, 64):
        raise RuntimeError(f"the row-split graph-LSTM cell serves 32 or 64 hidden channels, not {cout}")
    return getattr(_lib.lib(), ("stmp_lstm_wide_rows_" if cout == 64 else "stmp_lstm_rows_") + what)


def lstm_rows_pack_weights(variant: int, n_ops: int, cin: int, wx, wh, bx, bh, bg):
    """(w (4 cout, nb), b (4 cout,)): the row-split LSTM cell's packed weights from the parameters' layout in one launch
    (stmp_lstm_rows_pack_weights, or stmp_lstm_wide_rows_pack_weights at cout = 64; cout = wh.size(-1)).  GConvLSTM: wx (4, n_ops+1, cout,
    cin), wh (4, n_ops+1, cout, cout), bx / bh (4, cout) or None; GCLSTM: wx (4, cin, cout) (the dense W_g), wh as above, bx None, bh
    (4, cout) or None.  bg (4, cout): the gates' own biases b_g."""
    wx, wh, bg = _f32c(wx, "wx"), _f32c(wh, "wh"), _f32c(bg, "bg")
    cout = wh.size(-1)
    want_x = (4, cin, cout) if variant == _lib.LSTM_GC else (4, n_ops + 1, cout, cin)
    if wx.shape != want_x or wh.shape != (4, n_ops + 1, cout, cout) or bg.shape != (4, cout):
        raise RuntimeError(f"lstm_rows_pack_weights: wx must be {want_x}, wh (4, n_ops+1, {cout}, {cout}) and bg (4, {cout})")
    bx = None if bx is None else _f32c(bx, "bx")
    bh = None if bh is None else _f32c(bh, "bh")
    w = torch.empty(4 * cout, lstm_rows_nb(variant, n_ops, cin, cout), device=wx.device, dtype=torch.float32)
    b = torch.empty(4 * cout, device=wx.device, dtype=torch.float32)
    with torch.cuda.device(wx.device):
        _lib.check(_lstm_rows_entry(cout, "pack_weights")(variant, n_ops, cin, _lib.ptr(wx), _lib.ptr(wh), _lib.ptr(bx), _lib.ptr(bh),
                                                          _lib.ptr(bg), _lib.ptr(w), _lib.ptr(b), _lib.stream_ptr()))
    return w, b


def lstm_rows_fwd(plan: GraphPlan, variant: int, n_ops: int, x: torch.Tensor, h: Optional[torch.Tensor], c: Optional[torch.Tensor],
                  w: torch.Tensor, b: torch.Tensor, peep: Optional[torch.Tensor], train: bool = False):
    """Row-split peephole graph-LSTM cell (stmp_lstm_rows_fwd, or stmp_lstm_wide_rows_fwd for packed weights of 256 rows) on one graph:
    x (N, cin), h and c (N, cout) or None (zeros) -> (H', C'), cout = w.size(0) / 4.  peep (3, cout) = w_c_i | w_c_f | w_c_o, or None.
    With `train`, returns (H', C', stash (4, N, cout), S) -- the operands of lstm_rows_bwd / lstm_rows_wgrad."""
    x, w, b = _f32c(x, "X"), _f32c(w, "w"), _f32c(b, "b")
    N, cin = x.shape
    co = w.size(0) // 4
    f32 = dict(device=x.device, dtype=torch.float32)
    hc = None if h is None else _f32c(h, "H")
    cc = None if c is None else _f32c(c, "C")
    pc = None if peep is None else _f32c(peep, "peep")
    hout, cout = torch.empty(N, co, **f32), torch.empty(N, co, **f32)
    st = S = None
    ld = lstm_rows_basis_ld(variant, n_ops, cin, co)
    if train:
        st = torch.empty(4, N, co, **f32)
        S = torch.empty(N, ld, **f32)
    with torch.cuda.device(x.device):
        _lib.check(_lstm_rows_entry(co, "fwd")(plan.handle, variant, n_ops, cin, _lib.ptr(x), _lib.ptr(hc), _lib.ptr(cc), _lib.ptr(w),
                                               _lib.ptr(b), _lib.ptr(pc), _lib.ptr(hout), _lib.ptr(cout), _lib.ptr(st), _lib.ptr(S), ld,
                                               _lib.stream_ptr()))
    return (hout, cout, st, S) if train else (hout, cout)


def lstm_rows_bwd(plan: GraphPlan, variant: int, n_ops: int, gh, gc, c, cn, stash, w, peep, want_dx: bool, want_dh: bool, want_dc: bool,
                  cin: int):
    """(dpre (2, N, 2 cout), dx (N, cin) or None, dh or None, dc or None, scratch) of the row-split LSTM cell (stmp_lstm_rows_bwd, or
    stmp_lstm_wide_rows_bwd when cn has 64 channels); gh / gc may be None.  The scratch carries the per-CTA peephole sums to
    lstm_rows_wgrad."""
    N, co = cn.shape
    f32 = dict(device=cn.device, dtype=torch.float32)
    gh = None if gh is None else _f32c(gh, "gH")
    gc = None if gc is None else _f32c(gc, "gC")
    scr = torch.empty(int(_lstm_rows_entry(co, "scratch_bytes")(plan.handle)) // 4, **f32)
    dpre = torch.empty(2, N, 2 * co, **f32)
    dx = torch.empty(N, cin, **f32) if want_dx else None
    dh = torch.empty(N, co, **f32) if want_dh else None
    dc = torch.empty(N, co, **f32) if want_dc else None
    with torch.cuda.device(cn.device):
        _lib.check(_lstm_rows_entry(co, "bwd")(plan.handle, variant, n_ops, cin, _lib.ptr(gh), _lib.ptr(gc), _lib.ptr(c), _lib.ptr(cn),
                                               _lib.ptr(stash), _lib.ptr(w), _lib.ptr(peep), _lib.ptr(scr), _lib.ptr(dpre), _lib.ptr(dx),
                                               _lib.ptr(dh), _lib.ptr(dc), _lib.stream_ptr()))
    return dpre, dx, dh, dc, scr


def lstm_rows_wgrad(variant: int, n_ops: int, cin: int, S, dpre, scratch, has_peep: bool):
    """(dw (4 cout, nb), dbp (7 cout,)): the packed weights' gradient and, in one vector, the summed biases' gradient dbp[:4 cout] and the
    peepholes' dbp[4 cout:] (left unwritten without peepholes) of the row-split LSTM cell, two launches; cout = dpre.size(2) / 2.  n_ops = 2
    (the two-operator basis at 32 channels) takes stmp_lstm_rows_wgrad2, which has no peepholes."""
    dev = S.device
    co = dpre.size(2) // 2
    dw = torch.empty(4 * co, lstm_rows_nb(variant, n_ops, cin, co), device=dev, dtype=torch.float32)
    dbp = torch.empty(7 * co, device=dev, dtype=torch.float32)
    if n_ops == 2:                     # the two-operator basis (LRGCN, two relations): its own contraction, no peepholes
        L = _lib.lib()
        ws = _wgrad_workspace(dev, L.stmp_lstm_rows_wgrad2_workspace_bytes, cin)
        with torch.cuda.device(dev):
            _lib.check(L.stmp_lstm_rows_wgrad2(cin, S.size(0), S.size(1), _lib.ptr(S), _lib.ptr(dpre), _lib.ptr(ws), _lib.ptr(dw),
                                               _lib.ptr(dbp), _lib.stream_ptr()))
        return dw, dbp
    ws = _wgrad_workspace(dev, _lstm_rows_entry(co, "wgrad_workspace_bytes"), variant, n_ops, cin)
    dpeep = dbp[4 * co:] if has_peep else None
    with torch.cuda.device(dev):
        _lib.check(_lstm_rows_entry(co, "wgrad")(variant, n_ops, cin, S.size(0), S.size(1), _lib.ptr(S), _lib.ptr(dpre), _lib.ptr(scratch),
                                                 _lib.ptr(ws), _lib.ptr(dw), _lib.ptr(dbp), _lib.ptr(dpeep), _lib.stream_ptr()))
    return dw, dbp


class _LstmRowsFn(torch.autograd.Function):
    """Training form of the row-split peephole graph-LSTM cell (32 or 64 hidden channels, from the packed weights).  forward =
    `stmp_lstm_rows_fwd` (`stmp_lstm_wide_rows_fwd`) with the stash and the weight-gradient basis
    (the inference launch, so (H', C') are bit-identical to the `no_grad` ones); backward = `stmp_lstm_rows_bwd` + `stmp_lstm_rows_wgrad`:
    dX (when x requires grad), dH / dC (when h / c are given and require grad) and the packed weights', summed biases' and peepholes'
    gradients, handed to `params` as blocks described by `spec` (see _spec_grads; the peepholes sit in the bias vector after its 4 cout
    entries).  Either output's gradient may be None."""

    @staticmethod
    def forward(ctx, plan, variant, n_ops, x, h, c, w, b, peep, spec, *params):
        ctx.set_materialize_grads(False)
        x = _f32c(x.detach(), "X")
        hc = None if h is None else _f32c(h.detach(), "H")
        cc = None if c is None else _f32c(c.detach(), "C")
        hout, cout, stash, S = lstm_rows_fwd(plan, variant, n_ops, x, hc, cc, w, b, peep, train=True)
        ctx.plan, ctx.variant, ctx.n_ops, ctx.spec, ctx.cin = plan, variant, n_ops, spec, x.size(1)
        ctx.has_h, ctx.shapes = hc is not None, [p.shape for p in params]
        ctx.save_for_backward(cc, cout, stash, S, w, peep)
        return hout, cout

    @staticmethod
    def backward(ctx, gH, gC):
        c, cn, stash, S, w, peep = ctx.saved_tensors
        nin = 10 + len(ctx.spec)
        if gH is None and gC is None:
            return (None,) * nin
        want_dh = ctx.has_h and ctx.needs_input_grad[4]
        want_dc = c is not None and ctx.needs_input_grad[5]
        dpre, dx, dh, dc, scr = lstm_rows_bwd(ctx.plan, ctx.variant, ctx.n_ops, gH, gC, c, cn, stash, w, peep, ctx.needs_input_grad[3],
                                              want_dh, want_dc, ctx.cin)
        grads = [None] * len(ctx.spec)
        if any(ctx.needs_input_grad[10:]):
            dw, dbp = lstm_rows_wgrad(ctx.variant, ctx.n_ops, ctx.cin, S, dpre, scr, peep is not None)
            grads = [g.reshape(shape) for g, shape in zip(_spec_grads(ctx.spec, dw, dbp), ctx.shapes)]
        return (None, None, None, dx, dh, dc, None, None, None, None, *grads)


def lstm_rows_train(plan: GraphPlan, variant: int, n_ops: int, x, h, c, w, b, peep, spec, params):
    """Differentiable (w.r.t. x, h, c and `params`, see _LstmRowsFn) row-split peephole graph-LSTM cell -> (H', C').  x (N, cin); h, c
    (N, cout) or None (zeros, no state gradient)."""
    return _LstmRowsFn.apply(plan, variant, n_ops, x, h, c, w, b, peep, tuple(spec), *params)


def ggc_rows_supported(plan: GraphPlan, num_layers: int, cin: int, channels: int) -> bool:
    return bool(_lib.lib().stmp_ggc_rows_supported(plan.handle, num_layers, cin, channels))


def _ggc_scratch(plan: GraphPlan, C: int, device) -> torch.Tensor:
    return torch.empty(int(_lib.lib().stmp_ggc_rows_scratch_bytes(plan.handle, C)) // 4, device=device, dtype=torch.float32)


def ggc_rows_fwd(plan: GraphPlan, x: torch.Tensor, W: torch.Tensor, w_ih, w_hh, b_ih, b_hh, train: bool = False):
    """GatedGraphConv on a gated plan (stmp_ggc_rows_fwd): x (N, cin) -> x^L (N, C), W (L, C, C), W_ih / W_hh (3C, C), b_ih / b_hh (3C,);
    L launches (L + 1 for max).  With `train`, returns (out, stash (L, 8, N, C)), the operand of ggc_rows_bwd / ggc_rows_wgrad."""
    x, W = _f32c(x, "X"), _f32c(W, "weight")
    w_ih, w_hh, b_ih, b_hh = (_f32c(t, n) for t, n in ((w_ih, "weight_ih"), (w_hh, "weight_hh"), (b_ih, "bias_ih"), (b_hh, "bias_hh")))
    L, C = W.size(0), W.size(-1)
    N, cin = x.shape
    f32 = dict(device=x.device, dtype=torch.float32)
    out = torch.empty(N, C, **f32)
    stash = torch.empty(L, 8, N, C, **f32) if train else None
    scr = None if train else _ggc_scratch(plan, C, x.device)
    with torch.cuda.device(x.device):
        _lib.check(_lib.lib().stmp_ggc_rows_fwd(plan.handle, L, cin, C, _lib.ptr(x), _lib.ptr(W), _lib.ptr(w_ih), _lib.ptr(w_hh),
                                                _lib.ptr(b_ih), _lib.ptr(b_hh), _lib.ptr(scr), _lib.ptr(out), _lib.ptr(stash),
                                                _lib.stream_ptr()))
    return (out, stash) if train else out


class _GgcRowsFn(torch.autograd.Function):
    """Training form of the row-split GatedGraphConv.  forward = `stmp_ggc_rows_fwd` with the stash (the inference launches, so the output
    is bit-identical to the `no_grad` one); backward = `stmp_ggc_rows_bwd` + `stmp_ggc_rows_wgrad`: dX (when X requires grad) and the
    gradients of W, W_ih, W_hh, b_ih and b_hh in their own layouts."""

    @staticmethod
    def forward(ctx, plan, x, W, w_ih, w_hh, b_ih, b_hh):
        W, w_ih, w_hh = (_f32c(t.detach(), "weight") for t in (W, w_ih, w_hh))
        out, stash = ggc_rows_fwd(plan, x.detach(), W, w_ih, w_hh, b_ih.detach(), b_hh.detach(), train=True)
        ctx.plan, ctx.cin = plan, x.size(1)
        ctx.save_for_backward(stash, W, w_ih, w_hh)
        return out

    @staticmethod
    def backward(ctx, gout):
        stash, W, w_ih, w_hh = ctx.saved_tensors
        plan, L, C, N = ctx.plan, W.size(0), W.size(-1), stash.size(2)
        dev = stash.device
        f32 = dict(device=dev, dtype=torch.float32)
        gout = _f32c(gout, "gout")
        dG = torch.empty(L, N, 4 * C, **f32)
        dM = torch.empty(L, N, C, **f32)
        dx = torch.empty(N, ctx.cin, **f32) if ctx.needs_input_grad[1] else None
        L_ = _lib.lib()
        with torch.cuda.device(dev):
            _lib.check(L_.stmp_ggc_rows_bwd(plan.handle, L, ctx.cin, C, _lib.ptr(gout), _lib.ptr(stash), _lib.ptr(W), _lib.ptr(w_ih),
                                            _lib.ptr(w_hh), _lib.ptr(_ggc_scratch(plan, C, dev)), _lib.ptr(dG), _lib.ptr(dM), _lib.ptr(dx),
                                            _lib.stream_ptr()))
        grads = [None] * 5
        if any(ctx.needs_input_grad[2:]):
            ws = _wgrad_workspace(dev, L_.stmp_ggc_rows_wgrad_workspace_bytes, L, C)
            grads = [torch.empty(L, C, C, **f32), torch.empty(3 * C, C, **f32), torch.empty(3 * C, C, **f32),
                     torch.empty(3 * C, **f32), torch.empty(3 * C, **f32)]
            with torch.cuda.device(dev):
                _lib.check(L_.stmp_ggc_rows_wgrad(plan.handle, L, C, _lib.ptr(stash), _lib.ptr(dG), _lib.ptr(dM), _lib.ptr(ws),
                                                  *(_lib.ptr(g) for g in grads), _lib.stream_ptr()))
        return (None, dx, *grads)


def ggc_rows_train(plan: GraphPlan, x, W, w_ih, w_hh, b_ih, b_hh) -> torch.Tensor:
    """Differentiable (w.r.t. x and the five parameters, see _GgcRowsFn) row-split GatedGraphConv: x (N, cin) -> x^L (N, C)."""
    return _GgcRowsFn.apply(plan, x, W, w_ih, w_hh, b_ih, b_hh)


def evolvegcn_rows_supported(plan: GraphPlan, channels: int) -> bool:
    return bool(_lib.lib().stmp_evolvegcn_rows_supported(plan.handle, channels))


def evolvegcn_rows_fwd(plan: GraphPlan, x: torch.Tensor, w_prev: torch.Tensor, w_ih, w_hh, b_ih, b_hh, p=None, train: bool = False):
    """One EvolveGCN step (stmp_evolvegcn_rows_fwd): x (N, C), w_prev (C, C), the GRU's W_ih / W_hh (3C, C) and b_ih / b_hh (3C,), p (C,)
    for -H or None for -O -> (out (N, C), w_new (C, C), perm (C,) int32 or None, score (C,) or None, stash (N, C) with `train`, else None).
    One launch for -O, two for -H."""
    x, w_prev = _f32c(x, "X"), _f32c(w_prev, "weight")
    w_ih, w_hh, b_ih, b_hh = (_f32c(t, n) for t, n in ((w_ih, "weight_ih"), (w_hh, "weight_hh"), (b_ih, "bias_ih"), (b_hh, "bias_hh")))
    N, C = x.shape
    f32 = dict(device=x.device, dtype=torch.float32)
    out, w_new = torch.empty(N, C, **f32), torch.empty(C, C, **f32)
    stash = torch.empty(N, C, **f32) if train else None
    perm = score = scr = None
    if p is not None:
        p = _f32c(p, "pooling weight")
        perm, score = torch.empty(C, device=x.device, dtype=torch.int32), torch.empty(C, **f32)
        scr = torch.empty(int(_lib.lib().stmp_evolvegcn_rows_scratch_bytes(plan.handle, C)), device=x.device, dtype=torch.uint8)
    with torch.cuda.device(x.device):
        _lib.check(_lib.lib().stmp_evolvegcn_rows_fwd(plan.handle, C, *(_lib.ptr(t) for t in (x, w_prev, w_ih, w_hh, b_ih, b_hh, p, scr, out,
                                                                                              w_new, perm, score, stash)),
                                                      _lib.stream_ptr()))
    return out, w_new, perm, score, stash


class _EvolveGCNRowsFn(torch.autograd.Function):
    """Training form of one EvolveGCN step -> (out, w_new).  forward = `stmp_evolvegcn_rows_fwd` with the stash Op x, kept in ctx (the
    inference launches, so the outputs are bit-identical to the `no_grad` ones); backward = `stmp_evolvegcn_rows_bwd` +
    `stmp_evolvegcn_rows_wgrad`: dX (when X requires grad) and the gradients of w_prev, the four GRU tensors and p.  Either output's
    gradient may be None; dL/dw_new enters the GRU backward with the convolution's."""

    @staticmethod
    def forward(ctx, plan, x, w_prev, w_ih, w_hh, b_ih, b_hh, p):
        ctx.set_materialize_grads(False)
        ts = [None if t is None else t.detach() for t in (x, w_prev, w_ih, w_hh, b_ih, b_hh, p)]
        ts = [None if t is None else _f32c(t, "operand") for t in ts]
        out, w_new, perm, score, stash = evolvegcn_rows_fwd(plan, *ts, train=True)
        ctx.plan = plan
        ctx.save_for_backward(*ts, perm, score, stash, w_new)
        return out, w_new

    @staticmethod
    def backward(ctx, gout, gw):
        x, w_prev, w_ih, w_hh, b_ih, b_hh, p, perm, score, stash, w_new = ctx.saved_tensors
        if gout is None and gw is None:
            return (None,) * 8
        plan, dev = ctx.plan, x.device
        N, C = x.shape
        f32 = dict(device=dev, dtype=torch.float32)
        gout = torch.zeros(N, C, **f32) if gout is None else _f32c(gout, "gout")
        gw = None if gw is None else _f32c(gw, "gout")
        dx = torch.empty(N, C, **f32) if ctx.needs_input_grad[1] else None
        grads = [torch.empty(C, C, **f32), torch.empty(3 * C, C, **f32), torch.empty(3 * C, C, **f32), torch.empty(3 * C, **f32),
                 torch.empty(3 * C, **f32)]
        dp = torch.empty(C, **f32) if p is not None else None
        L_ = _lib.lib()
        ws = torch.empty(int(L_.stmp_evolvegcn_rows_workspace_bytes(plan.handle, C)), device=dev, dtype=torch.uint8)
        with torch.cuda.device(dev):
            _lib.check(L_.stmp_evolvegcn_rows_bwd(plan.handle, C, _lib.ptr(gout), _lib.ptr(stash), _lib.ptr(w_new), _lib.ptr(ws),
                                                  _lib.ptr(dx), _lib.stream_ptr()))
            _lib.check(L_.stmp_evolvegcn_rows_wgrad(plan.handle, C, _lib.ptr(ws), *(_lib.ptr(t) for t in (gw, x, w_prev, w_ih, w_hh, b_ih,
                                                                                                          b_hh, p, perm, score, *grads, dp,
                                                                                                          dx)),
                                                    _lib.stream_ptr()))
        want = ctx.needs_input_grad
        return (None, dx, *(g if want[2 + i] else None for i, g in enumerate(grads)), dp if p is not None and want[7] else None)


def evolvegcn_rows_train(plan: GraphPlan, x, w_prev, w_ih, w_hh, b_ih, b_hh, p=None):
    """Differentiable (w.r.t. x, w_prev, the GRU's four tensors and p, see _EvolveGCNRowsFn) EvolveGCN step -> (out (N, C), w_new (C, C))."""
    return _EvolveGCNRowsFn.apply(plan, x, w_prev, w_ih, w_hh, b_ih, b_hh, p)


def mpnn_rows_supported(plan: GraphPlan, cin: int, hidden: int, window: int) -> bool:
    return bool(_lib.lib().stmp_mpnn_rows_supported(plan.handle, cin, hidden, window))


def _mpnn_params(conv1, conv2, bn1, bn2, lstm1, lstm2):
    """The 17 tensors one MPNN-LSTM call reads, in the order of _MpnnRowsFn's inputs."""
    return (conv1.lin.weight, conv1.bias, conv2.lin.weight, conv2.bias, bn1.weight, bn1.bias, bn2.weight, bn2.bias,
            *(getattr(m, k) for m in (lstm1, lstm2) for k in ("weight_ih_l0", "weight_hh_l0", "bias_ih_l0", "bias_hh_l0")))


def mpnn_rows_fwd(plan: GraphPlan, x: torch.Tensor, num_nodes: int, window: int, conv1, conv2, bn1, bn2, lstm1, lstm2, training: bool,
                  p: float, u: Optional[torch.Tensor], params=None, train: bool = False):
    """The MPNN-LSTM forward (stmp_mpnn_rows_fwd, three launches): x (R, cin) with R = B * window * num_nodes -> (B num_nodes,
    64 + cin + window - 1) = [h1 | h2 | S].  conv1 / conv2 hold GCNConv's `lin.weight` (32, K) and `bias` (32); bn1 / bn2 are
    BatchNorm1d(32) modules (affine, running statistics tracked; updated in place when `training`, BatchNorm's mode); lstm1 / lstm2
    torch.nn.LSTM(64, 32) and (32, 32).  u (2, R, 32) holds the dropout uniforms (kept where u >= p) or None for no dropout.  `params`
    overrides the 16 tensors of _mpnn_params.  Returns out, or (out, scratch, stash) with `train` (the backward's operands).  No
    autograd."""
    x = _f32c(x, "X")
    R, cin = x.shape
    ts = [_f32c(t.detach(), "MPNN-LSTM parameter") for t in (params or _mpnn_params(conv1, conv2, bn1, bn2, lstm1, lstm2))]
    bns = []
    for bn, (w, b) in ((bn1, ts[4:6]), (bn2, ts[6:8])):
        mom = -1.0 if bn.momentum is None else float(bn.momentum)
        bns.append(([_lib.ptr(w), _lib.ptr(b), _lib.ptr(bn.running_mean), _lib.ptr(bn.running_var), _lib.ptr(bn.num_batches_tracked)],
                    float(bn.eps), mom))
    if u is not None:
        u = _f32c(u, "dropout uniforms")
        _require_numel("mpnn_rows_fwd", 2 * R * 32, u=u)
    out = torch.empty(R // window, 64 + cin + window - 1, device=x.device, dtype=torch.float32)
    L_ = _lib.lib()
    byt = lambda n: torch.empty(int(n), device=x.device, dtype=torch.uint8)
    scr = byt(L_.stmp_mpnn_rows_scratch_bytes(plan.handle, cin, 32, window))
    stash = byt(L_.stmp_mpnn_rows_stash_bytes(plan.handle, cin, 32, window)) if train else None
    with torch.cuda.device(x.device):
        _lib.check(L_.stmp_mpnn_rows_fwd(plan.handle, cin, 32, window, num_nodes, _lib.ptr(x), *(_lib.ptr(t) for t in ts[:4]), *bns[0][0],
                                         bns[0][1], bns[0][2], *bns[1][0], bns[1][1], bns[1][2], *(_lib.ptr(t) for t in ts[8:]),
                                         int(training), float(p), _lib.ptr(u), _lib.ptr(scr), _lib.ptr(stash), _lib.ptr(out),
                                         _lib.stream_ptr()))
    return (out, scr, stash) if train else out


class _MpnnRowsFn(torch.autograd.Function):
    """Training form of one MPNN-LSTM call.  forward = stmp_mpnn_rows_fwd with the stash (the inference launches: the outputs are
    bit-identical to the no_grad ones for the same mode and masks), scratch and stash kept in ctx; backward = stmp_mpnn_rows_bwd +
    stmp_mpnn_rows_wgrad: dX (when X requires grad) and the gradients of the 16 parameters."""

    @staticmethod
    def forward(ctx, plan, meta, x, *params):
        num_nodes, window, mods, training, p, u = meta
        out, scr, stash = mpnn_rows_fwd(plan, x.detach(), num_nodes, window, *mods, training, p, u, params=params, train=True)
        ctx.plan, ctx.meta, ctx.scr, ctx.stash = plan, (num_nodes, window, training, p if u is not None else 0.0), scr, stash
        ctx.save_for_backward(*(t.detach() for t in params))
        ctx.shape = x.shape
        return out

    @staticmethod
    def backward(ctx, gout):
        ps = [_f32c(t, "MPNN-LSTM parameter") for t in ctx.saved_tensors]
        num_nodes, window, training, p = ctx.meta
        R, cin = ctx.shape
        dev = gout.device
        gout = _f32c(gout, "gout")
        f32 = dict(device=dev, dtype=torch.float32)
        dx = torch.empty(R, cin, **f32) if ctx.needs_input_grad[2] else None
        dbn, dw, db = torch.empty(4, 32, **f32), torch.empty(320, 96, **f32), torch.empty(320, **f32)
        L_, h = _lib.lib(), ctx.plan.handle
        ws = torch.empty(int(L_.stmp_mpnn_rows_workspace_bytes(h, cin, 32, window)), device=dev, dtype=torch.uint8)
        with torch.cuda.device(dev):
            _lib.check(L_.stmp_mpnn_rows_bwd(h, cin, 32, window, num_nodes, _lib.ptr(gout), *(_lib.ptr(ps[i]) for i in (0, 2, 4, 6, 8, 9, 12,
                                                                                                                      13)),
                                             int(training), float(p), _lib.ptr(ctx.scr), _lib.ptr(ctx.stash), _lib.ptr(ws), _lib.ptr(dx),
                                             _lib.ptr(dbn), _lib.stream_ptr()))
            _lib.check(L_.stmp_mpnn_rows_wgrad(h, cin, 32, window, _lib.ptr(ctx.stash), _lib.ptr(ws), _lib.ptr(dw), _lib.ptr(db),
                                               _lib.stream_ptr()))
        ld1 = (cin + 7) // 8 * 8
        grads = (dw[256:288, :cin], db[256:288], dw[288:320, ld1:ld1 + 32], db[288:320], dbn[1], dbn[0], dbn[3], dbn[2],
                 dw[0:128, :64], dw[0:128, 64:96], db[0:128], db[0:128].clone(), dw[128:256, :32], dw[128:256, 32:64], db[128:256],
                 db[128:256].clone())
        want = ctx.needs_input_grad
        return (None, None, dx, *(g if want[3 + i] else None for i, g in enumerate(grads)))


def mpnn_rows_train(plan: GraphPlan, x, num_nodes: int, window: int, conv1, conv2, bn1, bn2, lstm1, lstm2, training: bool, p: float,
                    u: Optional[torch.Tensor]) -> torch.Tensor:
    """Differentiable (w.r.t. x and the 16 parameters of _mpnn_params, see _MpnnRowsFn) MPNN-LSTM call; arguments as mpnn_rows_fwd."""
    mods = (conv1, conv2, bn1, bn2, lstm1, lstm2)
    return _MpnnRowsFn.apply(plan, (num_nodes, window, mods, training, p, u), x, *_mpnn_params(*mods))


def agcrn_supported(batch: int, num_nodes: int, in_channels: int, out_channels: int, K: int, embedding_dimensions: int) -> bool:
    return bool(_lib.lib().stmp_agcrn_supported(batch, num_nodes, in_channels, out_channels, K, embedding_dimensions))


def _agcrn_dims(x, e, h, wp_gate, bp_gate, wp_update, bp_update):
    """(B, N, in, out, K, d) of one AGCRN call; raises on operands whose shapes disagree (the kernels trust them)."""
    B, N, cin = x.shape
    d, K, ci, out = wp_update.shape
    want = dict(e=(N, d), wp_gate=(d, K, ci, 2 * out), bp_gate=(d, 2 * out), bp_update=(d, out))
    got = dict(e=tuple(e.shape), wp_gate=tuple(wp_gate.shape), bp_gate=tuple(bp_gate.shape), bp_update=tuple(bp_update.shape))
    if h is not None:
        want["h"], got["h"] = (B, N, out), tuple(h.shape)
    if ci != cin + out or got != want:
        raise RuntimeError(f"agcrn: operand shapes {got} with X {tuple(x.shape)} and weights_pool {tuple(wp_update.shape)}, want {want}")
    return B, N, cin, out, K, d


def agcrn_fwd(x, e, h, wp_gate, bp_gate, wp_update, bp_update, train: bool = False):
    """One AGCRN call (stmp_agcrn_fwd, six launches, seven at K = 3): x (B, N, in), e (N, d), h (B, N, out) or None (zeros), the
    gate's pools (d, K, in + out, 2 out), (d, 2 out) and the update's (d, K, in + out, out), (d, out) -> H' (B, N, out).  Returns H',
    or (H', scratch, stash) with `train` (the backward's operands).  No autograd."""
    x, e, wp_gate, bp_gate, wp_update, bp_update = (_f32c(t.detach(), n) for t, n in (
        (x, "X"), (e, "E"), (wp_gate, "weights_pool"), (bp_gate, "bias_pool"), (wp_update, "weights_pool"), (bp_update, "bias_pool")))
    h = None if h is None else _f32c(h.detach(), "H")
    B, N, cin, out, K, d = _agcrn_dims(x, e, h, wp_gate, bp_gate, wp_update, bp_update)
    hout = torch.empty(B, N, out, device=x.device, dtype=torch.float32)
    L_ = _lib.lib()
    byt = lambda n: torch.empty(int(n), device=x.device, dtype=torch.uint8)
    scr = byt(L_.stmp_agcrn_scratch_bytes(B, N, cin, out, K))
    stash = byt(L_.stmp_agcrn_stash_bytes(B, N, cin, out, K)) if train else None
    with torch.cuda.device(x.device):
        _lib.check(L_.stmp_agcrn_fwd(B, N, cin, out, K, d, *(_lib.ptr(t) for t in (x, e, h, wp_gate, bp_gate, wp_update, bp_update, scr,
                                                                                  stash, hout)), _lib.stream_ptr()))
    return (hout, scr, stash) if train else hout


class _AgcrnFn(torch.autograd.Function):
    """Training form of one AGCRN call.  forward = stmp_agcrn_fwd with the stash (the inference launches, so H' is bit-identical to the
    no_grad call), scratch and stash kept in ctx; backward = stmp_agcrn_bwd: the gradients of X, E, H and both AVWGCNs' pools that
    autograd asks for."""

    @staticmethod
    def forward(ctx, x, e, h, wp_gate, bp_gate, wp_update, bp_update):
        ops_in = (x, e, h, wp_gate, bp_gate, wp_update, bp_update)
        hout, ctx.scr, ctx.stash = agcrn_fwd(*ops_in, train=True)
        ctx.save_for_backward(*(None if t is None else t.detach() for t in ops_in))
        return hout

    @staticmethod
    def backward(ctx, gout):
        x, e, h, wp_gate, bp_gate, wp_update, bp_update = (None if t is None else t.contiguous() for t in ctx.saved_tensors)
        B, N, cin, out, K, d = _agcrn_dims(x, e, h, wp_gate, bp_gate, wp_update, bp_update)
        gout = _f32c(gout, "gout")
        want = ctx.needs_input_grad
        new = lambda t, i: torch.empty_like(t) if want[i] and t is not None else None
        dx, de, dh, *dpools = (new(t, i) for i, t in enumerate((x, e, h, wp_gate, bp_gate, wp_update, bp_update)))
        L_ = _lib.lib()
        ws = torch.empty(int(L_.stmp_agcrn_workspace_bytes(B, N, cin, out, K)), device=x.device, dtype=torch.uint8)
        with torch.cuda.device(x.device):
            _lib.check(L_.stmp_agcrn_bwd(B, N, cin, out, K, d, *(_lib.ptr(t) for t in (x, e, h, wp_gate, bp_gate, wp_update, bp_update,
                                                                                      ctx.scr, ctx.stash, gout, ws, dx, dh, de, *dpools)),
                                         _lib.stream_ptr()))
        return (dx, de, dh, *dpools)


def agcrn_train(x, e, h, wp_gate, bp_gate, wp_update, bp_update) -> torch.Tensor:
    """Differentiable (w.r.t. x, e, h and the four pools, see _AgcrnFn) AGCRN call; arguments as agcrn_fwd."""
    return _AgcrnFn.apply(x, e, h, wp_gate, bp_gate, wp_update, bp_update)


def gman_attn_supported(batch: int, other: int, heads: int, width: int, Lq: int, Lk: int, spatial: bool, mask: bool) -> bool:
    """stmp_gman_attn_supported for one GMAN attention call: spatial (B, T = other, N = Lq = Lk) on the long kernel, else (B, Lq / Lk
    steps, N = other) on the short one."""
    return bool(_lib.lib().stmp_gman_attn_supported(batch, other, heads, width, Lq, Lk, int(mask), int(spatial)))


def _gman_problem(t: torch.Tensor, spatial: bool):
    """(p0, p1, sequence length) and the (s0, s1, sl) strides of a channels-last (B, T, N, D) operand: problems (b, t) over the nodes
    for the spatial attention, (b, n) over the steps otherwise."""
    if spatial:
        return (t.shape[0], t.shape[1], t.shape[2]), (t.stride(0), t.stride(1), t.stride(2))
    return (t.shape[0], t.shape[2], t.shape[1]), (t.stride(0), t.stride(2), t.stride(1))


def _gman_call(q, k, v, heads: int, width: int, spatial: bool, mask: bool):
    """The arguments every stmp_gman_attn_* call shares, with O's (B, Lq, N, D) layout; raises on operands whose shapes disagree."""
    if q.dim() != 4 or k.shape != v.shape or k.dim() != 4 or q.shape[-1] != heads * width or k.shape[-1] != heads * width or \
            q.shape[0] != k.shape[0] or (q.shape[2] != k.shape[2] if not spatial else q.shape[:3] != k.shape[:3]):
        raise RuntimeError(f"gman_attention: Q {tuple(q.shape)}, K {tuple(k.shape)}, V {tuple(v.shape)} with {heads} heads of width "
                           f"{width}")
    (p0, p1, lq), sq = _gman_problem(q, spatial)
    (_, _, lk), sk = _gman_problem(k, spatial)
    _, sv = _gman_problem(v, spatial)
    _, so = _gman_problem(torch.empty(q.shape, device="meta"), spatial)
    strides = (ctypes.c_int64 * 12)(*sq, *sk, *sv, *so)
    return (p0, p1, heads, width, lq, lk, int(mask), int(spatial)), strides


def gman_attn_fwd(q, k, v, heads: int, width: int, scale: float, spatial: bool, mask: bool, train: bool = False):
    """One GMAN attention (stmp_gman_attn_fwd, one launch): q (B, Lq, N, D), k and v (B, Lk, N, D), D = heads width, head h in channels
    [h width, (h + 1) width); spatial attends over the nodes (Lq = Lk), otherwise over the steps (mask: the reference's tril mask).
    Returns O (B, Lq, N, D), or (O, stash) with `train`.  No autograd."""
    q, k, v = (_f32c(t.detach(), n) for t, n in ((q, "Q"), (k, "K"), (v, "V")))
    dims, strides = _gman_call(q, k, v, heads, width, spatial, mask)
    o = torch.empty(q.shape, device=q.device, dtype=torch.float32)
    L_ = _lib.lib()
    stash = torch.empty(int(L_.stmp_gman_attn_stash_bytes(*dims[:3], dims[4])) // 4, device=q.device, dtype=torch.float32) \
        if train else None
    with torch.cuda.device(q.device):
        _lib.check(L_.stmp_gman_attn_fwd(*dims, scale, strides, *(_lib.ptr(t) for t in (q, k, v, o, stash)), _lib.stream_ptr()))
    return (o, stash) if train else o


class _GmanAttnFn(torch.autograd.Function):
    """Training form of one GMAN attention.  forward = stmp_gman_attn_fwd with the log-sum-exp stash (the inference launch, so O is
    bit-identical to the no_grad call), the stash kept in ctx; backward = stmp_gman_attn_bwd: the gradients of Q, K and V that autograd
    asks for, P recomputed from the stash."""

    @staticmethod
    def forward(ctx, q, k, v, heads, width, scale, spatial, mask):
        o, ctx.stash = gman_attn_fwd(q, k, v, heads, width, scale, spatial, mask, train=True)
        ctx.meta = (heads, width, scale, spatial, mask)
        ctx.save_for_backward(q.detach(), k.detach(), v.detach(), o)
        return o

    @staticmethod
    def backward(ctx, gout):
        q, k, v, o = (t.contiguous() for t in ctx.saved_tensors)
        heads, width, scale, spatial, mask = ctx.meta
        gout = _f32c(gout, "gout")
        dims, strides = _gman_call(q, k, v, heads, width, spatial, mask)
        want = ctx.needs_input_grad
        dq, dk, dv = (torch.empty_like(t) if want[i] else None for i, t in enumerate((q, k, v)))
        L_ = _lib.lib()
        ws = torch.empty(int(L_.stmp_gman_attn_workspace_bytes(*dims[:3], dims[4], dims[7])), device=q.device, dtype=torch.uint8)
        with torch.cuda.device(q.device):
            _lib.check(L_.stmp_gman_attn_bwd(*dims, scale, strides, *(_lib.ptr(t) for t in (q, k, v, o, ctx.stash, gout, ws, dq, dk, dv)),
                                             _lib.stream_ptr()))
        return dq, dk, dv, None, None, None, None, None


def gman_attention(q, k, v, heads: int, width: int, scale: float, spatial: bool, mask: bool, train: bool):
    """One GMAN attention on the fused kernels, differentiable w.r.t. q, k, v with `train` (see _GmanAttnFn); arguments as
    gman_attn_fwd."""
    if train:
        return _GmanAttnFn.apply(q, k, v, heads, width, scale, spatial, mask)
    return gman_attn_fwd(q, k, v, heads, width, scale, spatial, mask)


def mtgnn_supported(n: int, k: int, dim: int, channels: int, depth: int, batch: int, steps: int) -> bool:
    """stmp_mtgnn_supported: whether MTGNN's graph build and propagation kernels take a graph of n nodes with k entries per row (or
    the widest row of a predefined A), embeddings of width dim, and (batch, channels, n, steps) activations at gcn_depth `depth`."""
    return _lib.lib().stmp_mtgnn_supported(n, k, dim, channels, depth, batch, steps) == _lib.STMP_OK


def _mtgnn_sizes(n: int, w: int):
    """Element counts of the pattern (int32), state and values (fp32) buffers of an N-node graph of row width w (include/stmp.h)."""
    return 3 * n * w + 2 * n + 1, n * w + 2 * n, 2 * n * w + 2 * n


def _mtgnn_require_graph(fn: str, n: int, w: int, pattern, vals, state=None):
    """Raises unless the graph buffers hold the counts the kernels index for n nodes of row width w: they trust (n, w)."""
    if pattern.dim() != 1:
        raise RuntimeError(f"{fn}: the pattern must be flat, got {pattern.dim()} dimensions")
    np_, ns, nv = _mtgnn_sizes(n, w)
    _require_numel(fn, np_, pattern=pattern)
    _require_numel(fn, nv, values=vals)
    _require_numel(fn, ns, state=state)
    if pattern.dtype != torch.int32:
        raise RuntimeError(f"{fn}: the pattern must be int32, got {pattern.dtype}")


def _mtgnn_buffers(n: int, w: int, device):
    np_, ns, nv = _mtgnn_sizes(n, w)
    return (torch.empty(np_, device=device, dtype=torch.int32), torch.empty(ns, device=device, dtype=torch.float32),
            torch.empty(nv, device=device, dtype=torch.float32))


def mtgnn_graph_fwd(m1: torch.Tensor, m2: torch.Tensor, k: int, alpha: float):
    """GraphConstructor's top-k graph from its node vectors m1, m2 (N, dim) (stmp_mtgnn_graph_fwd, four launches):
    -> (pattern, state, values), see include/stmp.h.  No autograd."""
    m1, m2 = _f32c(m1.detach(), "M1"), _f32c(m2.detach(), "M2")
    n, dim = m1.shape
    if k > n:
        raise RuntimeError("selected index k out of range")
    pattern, state, vals = _mtgnn_buffers(n, k, m1.device)
    L_ = _lib.lib()
    ws = torch.empty(int(L_.stmp_mtgnn_graph_workspace_bytes(n)), device=m1.device, dtype=torch.uint8)
    with torch.cuda.device(m1.device):
        _lib.check(L_.stmp_mtgnn_graph_fwd(n, k, dim, alpha, *(_lib.ptr(t) for t in (m1, m2, ws, pattern, state, vals)), _lib.stream_ptr()))
    return pattern, state, vals


def mtgnn_graph_dense(A: torch.Tensor):
    """The same structures from the nonzeros of a predefined dense (N, N) A (stmp_mtgnn_graph_dense): -> (pattern, state, values, w)
    with w the widest row.  A setup path: sizing it reads one number back to the host."""
    A = _f32c(A.detach(), "A_tilde")
    n = A.shape[0]
    w = max(1, int((A != 0).sum(1).max().item()))
    pattern, state, vals = _mtgnn_buffers(n, w, A.device)
    L_ = _lib.lib()
    ws = torch.empty(int(L_.stmp_mtgnn_graph_workspace_bytes(n)), device=A.device, dtype=torch.uint8)
    with torch.cuda.device(A.device):
        _lib.check(L_.stmp_mtgnn_graph_dense(n, w, *(_lib.ptr(t) for t in (A, ws, pattern, state, vals)), _lib.stream_ptr()))
    return pattern, state, vals, w


class _MtgnnGraphFn(torch.autograd.Function):
    """(M1, M2) -> the operator values on the top-k pattern; the pattern is a non-differentiable second output.  backward =
    stmp_mtgnn_graph_bwd: both normalisations, the mask, relu and tanh, then dM1 = (dz - dz^T) M2, dM2 = (dz^T - dz) M1."""

    @staticmethod
    def forward(ctx, m1, m2, k, alpha):
        pattern, state, vals = mtgnn_graph_fwd(m1, m2, k, alpha)
        ctx.meta = (k, alpha)
        ctx.save_for_backward(m1.detach().contiguous(), m2.detach().contiguous(), pattern, state, vals)
        ctx.mark_non_differentiable(pattern)
        return vals, pattern

    @staticmethod
    def backward(ctx, dvals, _dpattern):
        m1, m2, pattern, state, vals = ctx.saved_tensors
        k, alpha = ctx.meta
        n, dim = m1.shape
        _mtgnn_require_graph("mtgnn_graph_bwd", n, k, pattern, dvals, state)
        dvals = _f32c(dvals, "dvals")
        dm1, dm2 = torch.empty_like(m1), torch.empty_like(m2)
        L_ = _lib.lib()
        ws = torch.empty(int(L_.stmp_mtgnn_graph_bwd_workspace_bytes(n)), device=m1.device, dtype=torch.uint8)
        with torch.cuda.device(m1.device):
            _lib.check(L_.stmp_mtgnn_graph_bwd(n, k, dim, alpha, *(_lib.ptr(t) for t in (m1, m2, pattern, state, vals, dvals, ws, dm1, dm2)),
                                               _lib.stream_ptr()))
        return dm1, dm2, None, None


def mtgnn_graph(m1: torch.Tensor, m2: torch.Tensor, k: int, alpha: float, train: bool):
    """The learned graph's (values, pattern); with `train` the values are differentiable w.r.t. m1 and m2 (_MtgnnGraphFn)."""
    if train:
        return _MtgnnGraphFn.apply(m1, m2, k, alpha)
    pattern, _, vals = mtgnn_graph_fwd(m1, m2, k, alpha)
    return vals, pattern


def mtgnn_prop_fwd(x: torch.Tensor, pattern: torch.Tensor, vals: torch.Tensor, w: int, depth: int, alpha: float) -> torch.Tensor:
    """Both MixProps' hop chains (stmp_mtgnn_prop_fwd, 2 depth launches): x (B, C, N, T) -> hops (B, 2 depth C, N, T)."""
    _mtgnn_require_graph("mtgnn_prop_fwd", x.shape[2], w, pattern, vals)
    x = _f32c(x.detach(), "X")
    B, C, N, T = x.shape
    hops = torch.empty(B, 2 * depth * C, N, T, device=x.device, dtype=torch.float32)
    with torch.cuda.device(x.device):
        _lib.check(_lib.lib().stmp_mtgnn_prop_fwd(B, C, N, T, w, depth, alpha, *(_lib.ptr(t) for t in (x, pattern, vals.detach(), hops)),
                                                  _lib.stream_ptr()))
    return hops


def _mixprop_weights(w1, w2, C: int):
    """The two MixProp MLPs as one: the X block's weights summed (both MLPs read H_0 = X), then operator 1's hops, operator 2's."""
    w1, w2 = w1.view(w1.shape[0], -1), w2.view(w2.shape[0], -1)
    return w1[:, :C] + w2[:, :C], torch.cat((w1[:, C:], w2[:, C:]), dim=1)


def _mixprop_out(x, hops, w1, b1, w2, b2):
    B, C, N, T = x.shape
    wx, wh = _mixprop_weights(w1, w2, C)
    y = torch.matmul(wh, hops.view(B, hops.shape[1], N * T))
    y += torch.matmul(wx, x.reshape(B, C, N * T))
    y += (b1 + b2).view(1, -1, 1)
    return y.view(B, wx.shape[0], N, T)


class _MtgnnMixPropFn(torch.autograd.Function):
    """mixprop1(X, A) + mixprop2(X, A^T) of one MTGNN layer: (X, values, MLP weights) -> output (B, C_out, N, T).  forward =
    stmp_mtgnn_prop_fwd and the MLPs as fp32 GEMMs; backward = the GEMMs' transposes, then stmp_mtgnn_prop_bwd (the adjoint hop chains
    into dX and, when asked for, the values' gradient)."""

    @staticmethod
    def forward(ctx, x, vals, w1, b1, w2, b2, pattern, w, depth, alpha):
        x = _f32c(x.detach(), "X")
        hops = mtgnn_prop_fwd(x, pattern, vals, w, depth, alpha)
        ctx.meta = (w, depth, alpha)
        ctx.save_for_backward(x, vals.detach(), w1.detach(), w2.detach(), hops, pattern)
        return _mixprop_out(x, hops, w1.detach(), b1.detach(), w2.detach(), b2.detach())

    @staticmethod
    def backward(ctx, gy):
        x, vals, w1, w2, hops, pattern = ctx.saved_tensors
        w, depth, alpha = ctx.meta
        B, C, N, T = x.shape
        gy = _f32c(gy, "gout").view(B, w1.shape[0], N * T)
        wx, wh = _mixprop_weights(w1, w2, C)
        want = ctx.needs_input_grad
        dx = torch.matmul(wx.t(), gy)
        dhops = torch.matmul(wh.t(), gy)
        dvals = torch.empty_like(vals) if want[1] else None
        with torch.cuda.device(x.device):
            _lib.check(_lib.lib().stmp_mtgnn_prop_bwd(B, C, N, T, w, depth, alpha,
                                                      *(_lib.ptr(t) for t in (x, pattern, vals, hops, dhops, dx, dvals)), _lib.stream_ptr()))
        dw1 = dw2 = db = None
        if want[2] or want[4]:
            dwx = torch.matmul(gy, x.view(B, C, N * T).transpose(1, 2)).sum(0)
            dwh = torch.matmul(gy, hops.view(B, hops.shape[1], N * T).transpose(1, 2)).sum(0)
            gC = depth * C
            dw1 = torch.cat((dwx, dwh[:, :gC]), dim=1).view_as(w1)
            dw2 = torch.cat((dwx, dwh[:, gC:]), dim=1).view_as(w2)
        if want[3] or want[5]:
            db = gy.sum((0, 2))
        return (dx.view(B, C, N, T) if want[0] else None, dvals, dw1, db, dw2, db, None, None, None, None)


def mtgnn_mixprop(x, vals, pattern, w: int, depth: int, alpha: float, w1, b1, w2, b2, train: bool) -> torch.Tensor:
    """One MTGNN layer's two MixProps over the graph (vals, pattern) of row width w, x (B, C, N, T): differentiable w.r.t. x, vals and
    the MLP weights with `train` (_MtgnnMixPropFn)."""
    if train:
        return _MtgnnMixPropFn.apply(x, vals, w1, b1, w2, b2, pattern, w, depth, alpha)
    x = _f32c(x.detach(), "X")
    return _mixprop_out(x, mtgnn_prop_fwd(x, pattern, vals, w, depth, alpha), w1.detach(), b1.detach(), w2.detach(), b2.detach())


def _tgcn_entry(co: int, name: str):
    """The library entry `name` of the fused TGCN kernels at hidden width `co`: stmp_tgcn_<name> at 32, stmp_tgcn_wide_<name> at 64."""
    if co not in (32, 64):
        raise RuntimeError(f"the fused TGCN kernels take 32 or 64 hidden channels, got {co}")
    return getattr(_lib.lib(), ("stmp_tgcn_" if co == 32 else "stmp_tgcn_wide_") + name)


def tgcn_attn_fwd(plan: GraphPlan, x: torch.Tensor, A: torch.Tensor, Bm: torch.Tensor, c: torch.Tensor,
                  probs: Optional[torch.Tensor] = None, h: Optional[torch.Tensor] = None, h_shared: bool = False) -> torch.Tensor:
    """Fused A3TGCN(2) / TGCN(2) forward (stmp_tgcn_attn_fwd at 32 hidden channels, stmp_tgcn_wide_attn_fwd at 64; the width Co is
    Bm.shape[0]).  x (B,N,Fin,P) -> (B,N,Co); h (B,N,Co), or (N,Co) with h_shared=True (the same state for every batch row), or None
    (zeros)."""
    x = _f32c(x, "X")
    if x.dim() != 4 or x.size(1) != plan.num_nodes:
        raise RuntimeError(f"X must be (B,{plan.num_nodes},Fin,P), got {tuple(x.shape)}")
    B, N, fin, P = x.shape
    A, Bm, c = _f32c(A, "A"), _f32c(Bm, "Bm"), _f32c(c, "c")
    co = Bm.shape[0]
    entry = _tgcn_entry(co, "attn_fwd")
    if A.shape != (fin, 3 * co) or Bm.shape != (co, 3 * co) or c.numel() != 3 * co:
        raise RuntimeError(f"folded weights must be A (Fin,{3 * co}), Bm ({co},{3 * co}), c ({3 * co},)")
    out = torch.empty((B, N, co), dtype=torch.float32, device=x.device)
    if B == 0:
        return out
    hc, hs = None, 0
    if h is not None:
        hc = _f32c(h, "H")
        hs = 0 if h_shared else N * co
    pr = None if probs is None else _f32c(probs.detach(), "probs")
    with torch.cuda.device(x.device):
        _lib.check(entry(plan.handle, B, fin, P, _lib.ptr(x), _lib.ptr(hc), hs, _lib.ptr(A), _lib.ptr(Bm), _lib.ptr(c), _lib.ptr(pr),
                         _lib.ptr(out), _lib.stream_ptr()))
    return out


class _TgcnAttnFn(torch.autograd.Function):
    """Training form of the fused A3TGCN(2) / TGCN(2) forward for H = None: forward = `stmp_tgcn_attn_fwd`, backward =
    `stmp_tgcn_attn_bwd` (gates recomputed, gradients of the folded weights A, c and of the attention probabilities reduced on the
    device; the *_wide_* entries at 64 hidden channels).  No gradient w.r.t. X."""

    @staticmethod
    def forward(ctx, plan, x, A, Bm, c, probs):
        out = tgcn_attn_fwd(plan, x, A.detach(), Bm.detach(), c.detach(), None if probs is None else probs.detach(), None)
        ctx.plan, ctx.has_probs, ctx.co = plan, probs is not None, Bm.shape[0]
        ctx.save_for_backward(x, A.detach(), c.detach(), probs.detach() if probs is not None else x.new_empty(0))
        return out

    @staticmethod
    def backward(ctx, gout):
        x, A, c, probs = ctx.saved_tensors
        plan, co = ctx.plan, ctx.co
        B, N, fin, P = x.shape
        gout = _f32c(gout, "gout")
        dev = x.device
        if B == 0:                                  # nothing to launch (empty tensors have NULL data pointers)
            return None, None, torch.zeros_like(A), None, torch.zeros_like(c), torch.zeros_like(probs) if ctx.has_probs else None
        ws = torch.empty(int(_tgcn_entry(co, "attn_bwd_workspace_bytes")(plan.handle, B)), dtype=torch.uint8, device=dev)
        dA = torch.empty(fin, 3 * co, dtype=torch.float32, device=dev)
        dc = torch.empty(3 * co, dtype=torch.float32, device=dev)
        dprobs = torch.empty(P, dtype=torch.float32, device=dev) if ctx.has_probs else None
        with torch.cuda.device(dev):
            _lib.check(_tgcn_entry(co, "attn_bwd")(plan.handle, B, fin, P, _lib.ptr(_f32c(x, "X")), _lib.ptr(_f32c(A, "A")),
                                                   _lib.ptr(_f32c(c, "c")), _lib.ptr(_f32c(probs, "probs")) if ctx.has_probs else None,
                                                   _lib.ptr(gout), _lib.ptr(ws), _lib.ptr(dA), _lib.ptr(dc), _lib.ptr(dprobs),
                                                   _lib.stream_ptr()))
        return None, None, dA, None, dc, dprobs


def tgcn_attn_train(plan: GraphPlan, x, A, Bm, c, probs=None) -> torch.Tensor:
    """Differentiable (w.r.t. A, c, probs) fused A3TGCN(2) / TGCN(2) forward for H = None."""
    return _TgcnAttnFn.apply(plan, x, A, Bm, c, probs)


class _TgcnCellFn(torch.autograd.Function):
    """Training form of one TGCN / TGCN2 cell step with an incoming state: forward = `stmp_tgcn_attn_fwd` (periods = 1, H given; the
    same launch as inference, so the output is bit-identical to it), backward = `stmp_tgcn_cell_bwd` (gates recomputed; dH and the
    gradients of the folded weights A, Bm, c; the *_wide_* entries at 64 hidden channels).  No gradient w.r.t. X."""

    @staticmethod
    def forward(ctx, plan, x, h, A, Bm, c):
        A, Bm, c, h = A.detach(), Bm.detach(), c.detach(), _f32c(h.detach(), "H")
        out = tgcn_attn_fwd(plan, x, A, Bm, c, None, h)
        ctx.plan = plan
        ctx.save_for_backward(x, h, A, Bm, c)
        return out

    @staticmethod
    def backward(ctx, gout):
        x, h, A, Bm, c = ctx.saved_tensors
        B, N, fin = x.shape[:3]
        co = Bm.shape[0]
        dev = x.device
        want_dh = ctx.needs_input_grad[2]
        dh = torch.empty(B, N, co, dtype=torch.float32, device=dev) if want_dh else None
        if B == 0:                                  # nothing to launch (empty tensors have NULL data pointers)
            return None, None, dh, torch.zeros_like(A), torch.zeros_like(Bm), torch.zeros_like(c)
        dA = torch.empty(fin, 3 * co, dtype=torch.float32, device=dev)
        dBm = torch.empty(co, 3 * co, dtype=torch.float32, device=dev)
        dc = torch.empty(3 * co, dtype=torch.float32, device=dev)
        gout = _f32c(gout, "gout")
        handle = ctx.plan.handle
        ws = torch.empty(int(_tgcn_entry(co, "cell_bwd_workspace_bytes")(handle, B)), dtype=torch.uint8, device=dev)
        with torch.cuda.device(dev):
            _lib.check(_tgcn_entry(co, "cell_bwd")(handle, B, fin, _lib.ptr(_f32c(x, "X")), _lib.ptr(h), N * co, _lib.ptr(A), _lib.ptr(Bm),
                                                   _lib.ptr(c), _lib.ptr(gout), _lib.ptr(ws), _lib.ptr(dh), _lib.ptr(dA), _lib.ptr(dBm),
                                                   _lib.ptr(dc), _lib.stream_ptr()))
        return None, None, dh, dA, dBm, dc


def tgcn_cell_train(plan: GraphPlan, x, h, A, Bm, c) -> torch.Tensor:
    """Differentiable (w.r.t. h, A, Bm, c) fused TGCN(2) cell step with an incoming state.  x (B,N,Fin,1), h (B,N,Co) -> (B,N,Co),
    Co = Bm.shape[0] = 32 or 64."""
    return _TgcnCellFn.apply(plan, x, h, A, Bm, c)


def spmm_cols(plan: GraphPlan, op: int, buf: torch.Tensor, src_col: int, dst_col: int, width: int, alpha: float = 1.0,
              z_col: Optional[int] = None, beta: float = 0.0, transposed: bool = False):
    """In-place column-block product inside one basis buffer `buf` (..., N, LD):
    buf[..., dst_col:dst_col+width] = alpha * A_op buf[..., src_col:+width] + beta * buf[..., z_col:+width].
    Lets T_k be written straight into its slot of S = [T_0 | T_1 | ...] (no torch.cat of large tensors); with
    `transposed` (A_op^T) and z_col == dst_col it is the accumulate step of the basis adjoint.  src and dst blocks must
    not overlap; z may alias dst exactly (each output element reads its own z before it is written)."""
    _require_cuda(buf, "buf")
    b3 = buf if buf.dim() == 3 else buf.unsqueeze(0)
    B, N, LD = b3.shape
    if not b3.is_contiguous() or N != plan.num_nodes:
        raise RuntimeError("basis buffer must be contiguous (..., N, LD)")
    base, es = b3.data_ptr(), 4
    pz = None if z_col is None else ctypes.c_void_p(base + z_col * es)
    with torch.cuda.device(buf.device):
        rc = _lib.lib().stmp_spmm(plan.handle, op, 1 if transposed else 0, B, width, ctypes.c_void_p(base + src_col * es), LD, N * LD,
                                  ctypes.c_void_p(base + dst_col * es), LD, N * LD, alpha, pz, LD, N * LD, beta, None,
                                  _lib.stream_ptr())
    _lib.check(rc)


def gemm_prepack(W: torch.Tensor) -> torch.Tensor:
    """Split a (K,N) fp32 weight into the packed fp16 hi/lo buffer of stmp_gemm_f32 (once per weight update)."""
    W = _f32c(W, "W")
    K, N = W.shape
    packed = torch.empty(int(_lib.lib().stmp_gemm_packed_elems(K, N)), dtype=torch.float16, device=W.device)
    with torch.cuda.device(W.device):
        _lib.check(_lib.lib().stmp_gemm_prepack(_lib.ptr(W), N, K, N, _lib.ptr(packed), _lib.stream_ptr()))
    return packed


def gemm(A: torch.Tensor, packed: torch.Tensor, K: int, N: int, bias: Optional[torch.Tensor] = None,
         out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """C = A @ W + bias on wgmma with the fp16 hi/lo operand split: fp32-class accuracy for |operands| between about 2^-3 and 2^15,
    an absolute floor of about 2^-25 per operand element below that (include/stmp.h, K4).  A (..., K) contiguous.
    `out`: a 2-D (M, N) view with unit column stride (e.g. a column block of a wider buffer) to write into."""
    A = _f32c(A, "A")
    M = A.numel() // K
    if out is None:
        C = torch.empty(*A.shape[:-1], N, dtype=torch.float32, device=A.device)
        ldc = N
    else:
        C = out
        if C.dim() != 2 or C.size(0) != M or C.size(1) != N or C.stride(1) != 1 or C.dtype != torch.float32:
            raise RuntimeError("gemm: `out` must be a float32 (M, N) view with unit column stride")
        ldc = C.stride(0)
    b = None if bias is None else _f32c(bias.detach(), "bias")
    with torch.cuda.device(A.device):
        _lib.check(_lib.lib().stmp_gemm_f32(_lib.ptr(A), K, M, K, N, _lib.ptr(packed), _lib.ptr(b), _lib.ptr(C), ldc, _lib.stream_ptr()))
    return C


EPI_BIAS, EPI_RELU, EPI_RELU_LN = 0, 1, 2


def _weight_image(packed: torch.Tensor, N: int, nblk: int) -> torch.Tensor:
    img = torch.empty(int(_lib.lib().stmp_gemm_blocks_image_bytes(N, nblk)), dtype=torch.uint8, device=packed.device)
    with torch.cuda.device(packed.device):
        _lib.check(_lib.lib().stmp_gemm_blocks_image(_lib.ptr(packed), N, nblk, _lib.ptr(img), _lib.stream_ptr()))
    return img


def gemm_blocks_prepack(blocks):
    """Pack the per-block weights [(width_i, N) fp32 ...] of a blocked GEMM: every block is zero-padded to 64 rows, the stack
    (nblk*64, N) is split into fp16 hi/lo (stmp_gemm_prepack) and rewritten as the per-k-block shared-memory image the kernel
    fetches by TMA (stmp_gemm_blocks_image).  Returns (packed, image)."""
    N = blocks[0].size(1)
    W = torch.zeros(64 * len(blocks), N, device=blocks[0].device, dtype=torch.float32)
    for i, w in enumerate(blocks):
        if w.size(0) > 64 or w.size(1) != N:
            raise RuntimeError("blocked GEMM: weight blocks must be (<=64, N)")
        W[64 * i:64 * i + w.size(0)] = w
    packed = gemm_prepack(W)
    return packed, _weight_image(packed, N, len(blocks))


def gemm_blocks(blocks, packed: torch.Tensor, N: int, ncols: int, bias: Optional[torch.Tensor] = None, epilogue: int = EPI_BIAS,
                gamma=None, beta=None, eps: float = 1e-5, seq: int = 1, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """C[m, :ncols] = epilogue(sum_i A_i[m + shift_i, :width_i] @ W_i + bias)  (stmp_gemm_blocks_f32).
    blocks: list of (tensor, width, shift): `tensor` is a 2-D fp32 CUDA view (M, >=width) with unit column stride."""
    M = blocks[0][0].size(0)
    dev = blocks[0][0].device
    n = len(blocks)
    ptrs = (ctypes.c_void_p * n)()
    lds = (ctypes.c_int64 * n)()
    widths = (ctypes.c_int32 * n)()
    shifts = (ctypes.c_int32 * n)()
    for i, (t, width, shift) in enumerate(blocks):
        _require_cuda(t, "block")
        if t.dtype != torch.float32 or t.dim() != 2 or t.size(0) != M or (t.size(1) > 1 and t.stride(1) != 1) or t.size(1) < width:
            raise RuntimeError("blocked GEMM: every block must be a float32 (M, >=width) view with unit column stride")
        ptrs[i], lds[i], widths[i], shifts[i] = t.data_ptr(), t.stride(0), width, shift
    C = torch.empty((M, ncols), dtype=torch.float32, device=dev) if out is None else out
    v = [None if t is None else _f32c(t.detach(), "param") for t in (bias, gamma, beta)]
    packed, image = packed if isinstance(packed, tuple) else (packed, None)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().stmp_gemm_blocks_f32(M, N, ncols, n, ctypes.cast(ptrs, ctypes.c_void_p), ctypes.cast(lds, ctypes.c_void_p),
                                                   ctypes.cast(widths, ctypes.c_void_p), ctypes.cast(shifts, ctypes.c_void_p), seq,
                                                   _lib.ptr(packed), _lib.ptr(image), _lib.ptr(v[0]), epilogue, _lib.ptr(v[1]), _lib.ptr(v[2]), eps,
                                                   _lib.ptr(C), C.stride(0), _lib.stream_ptr()))
    return C


def astgcn_factors(Xc, U1, U2, U3, be, Ve, W1, W2, W3, want_E: bool = False):
    """(lhs_s (B,N,T), rhs_s (B,T,N) [, E (B,T,T)]) of an ASTGCN block from channels-last X (B,N,T,F): temporal attention, X~ = X E and
    the spatial-attention factors in one launch (stmp_astgcn_factors_fwd)."""
    Xc = _f32c(Xc, "X")
    B, N, T, Fi = Xc.shape
    lhs = torch.empty((B, N, T), dtype=torch.float32, device=Xc.device)
    rhs = torch.empty((B, T, N), dtype=torch.float32, device=Xc.device)
    E = torch.empty((B, T, T), dtype=torch.float32, device=Xc.device) if want_E else None
    v = [_f32c(t.detach(), "param") for t in (U1, U2, U3, be.reshape(T, T), Ve, W1, W2, W3)]
    with torch.cuda.device(Xc.device):
        _lib.check(_lib.lib().stmp_astgcn_factors_fwd(B, N, T, Fi, _lib.ptr(Xc), *[_lib.ptr(t) for t in v], _lib.ptr(lhs), _lib.ptr(rhs),
                                                      _lib.ptr(E), _lib.stream_ptr()))
    return (lhs, rhs, E) if want_E else (lhs, rhs)


def spatial_attention_prepack(Vs: torch.Tensor) -> torch.Tensor:
    """Vs (N,N) -> packed fp16 hi/lo of Vs^T zero-padded to (P,P), P = N rounded up to 64."""
    n = Vs.size(0)
    P = (n + 63) // 64 * 64
    W = torch.zeros(P, P, device=Vs.device, dtype=torch.float32)
    W[:n, :n] = Vs.detach().t()
    packed = gemm_prepack(W)
    return packed, _weight_image(packed, P, P // 64)


SPATT_ONE_TILE_MAX = 320     # widest padded node count stmp_spatial_attention_fwd holds in one CTA row tile


def _spatt_factors(lhs, rhs, bsT):
    """Contiguous fp32 factors; an lhs view that does not start on 16 bytes is copied (both kernels read its 48-byte rows as float4 at T = 12)."""
    lhs, rhs, bsT = _f32c(lhs, "lhs"), _f32c(rhs, "rhs"), _f32c(bsT, "bsT")
    if lhs.data_ptr() % 16:
        lhs = lhs.clone()
    return lhs, rhs, bsT


def spatial_attention(lhs: torch.Tensor, rhs: torch.Tensor, bsT: torch.Tensor, vsT_packed: torch.Tensor) -> torch.Tensor:
    """ST (B, N, P) with ST[b, j, i] = softmax_dim1(Vs @ sigmoid(lhs @ rhs + bs))[b, i, j]; columns >= N are zero.
    P = N rounded up to 64 <= 320: one kernel (stmp_spatial_attention_fwd); up to 1024 nodes: the column-tiled pair (spatial_attention_tiled)."""
    P = (lhs.size(1) + 63) // 64 * 64
    if P > SPATT_ONE_TILE_MAX:
        return spatial_attention_tiled(lhs, rhs, bsT, vsT_packed)
    lhs, rhs, bsT = _spatt_factors(lhs, rhs, bsT)
    B, n, T = lhs.shape
    st = torch.empty((B, n, P), dtype=torch.float32, device=lhs.device)
    packed, image = vsT_packed if isinstance(vsT_packed, tuple) else (vsT_packed, None)
    with torch.cuda.device(lhs.device):
        _lib.check(_lib.lib().stmp_spatial_attention_fwd(B, n, T, _lib.ptr(lhs), _lib.ptr(rhs), _lib.ptr(bsT), _lib.ptr(packed),
                                                         _lib.ptr(image), _lib.ptr(st), P, _lib.stream_ptr()))
    return st


def spatial_attention_tiled(lhs: torch.Tensor, rhs: torch.Tensor, bsT: torch.Tensor, vsT_packed) -> torch.Tensor:
    """`spatial_attention` on the column-tiled kernel pair (stmp_spatial_attention_tiled_fwd), any 1 <= N <= 1024; the per-row softmax
    statistics go to a workspace from the caching allocator, so the call is capturable."""
    lhs, rhs, bsT = _spatt_factors(lhs, rhs, bsT)
    B, n, T = lhs.shape
    P = (n + 63) // 64 * 64
    st = torch.empty((B, n, P), dtype=torch.float32, device=lhs.device)
    packed = vsT_packed[0] if isinstance(vsT_packed, tuple) else vsT_packed
    l = _lib.lib()
    nbytes = max(int(l.stmp_spatial_attention_tiled_workspace_bytes(B, n)), 0)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=lhs.device)
    with torch.cuda.device(lhs.device):
        _lib.check(l.stmp_spatial_attention_tiled_fwd(B, n, T, _lib.ptr(lhs), _lib.ptr(rhs), _lib.ptr(bsT), _lib.ptr(packed), _lib.ptr(st), P,
                                                      _lib.ptr(ws), nbytes, _lib.stream_ptr()))
    return st


def spmm_attT(plan: GraphPlan, op: int, x: torch.Tensor, attT: torch.Tensor, alpha: float = 1.0) -> torch.Tensor:
    """y = alpha * (A_op * att) x with the attention given transposed / row-padded (B, N, ld) as `spatial_attention` writes it."""
    x = _f32c(x, "x")
    B, N, F = x.shape
    y = torch.empty_like(x)
    with torch.cuda.device(x.device):
        _lib.check(_lib.lib().stmp_spmm_att_t(plan.handle, op, B, F, _lib.ptr(x), F, N * F, _lib.ptr(y), F, N * F, alpha, None, F, N * F, 0.0,
                                             _lib.ptr(attT), attT.stride(1), _lib.stream_ptr()))
    return y


def gemm_lstm(A: torch.Tensor, packed: torch.Tensor, K: int, cout: int, conv_bias, cell, wci, wcf, wco, bi, bf, bc, bo):
    """(H', C') = peephole-LSTM gates of (A @ W + conv_bias), fused in the GEMM epilogue (stmp_gemm_lstm_f32).  The kernel walks the
    M = A.numel() / K rows of A, reading and writing one state row per row of A."""
    M = A.numel() // K
    _require_numel("gemm_lstm", M * K, A=A)
    _require_numel("gemm_lstm", M * cout, cell=cell)
    _require_numel("gemm_lstm", 4 * cout, conv_bias=conv_bias)
    _require_numel("gemm_lstm", cout, wci=wci, wcf=wcf, wco=wco, bi=bi, bf=bf, bc=bc, bo=bo)
    A, cell = _f32c(A, "A"), _f32c(cell, "C")
    h = torch.empty_like(cell)
    c = torch.empty_like(cell)
    v = [None if t is None else _f32c(t.detach().reshape(-1), "param") for t in (conv_bias, wci, wcf, wco, bi, bf, bc, bo)]
    with torch.cuda.device(A.device):
        _lib.check(_lib.lib().stmp_gemm_lstm_f32(_lib.ptr(A), K, M, K, cout, _lib.ptr(packed), _lib.ptr(v[0]), _lib.ptr(cell),
                                                 _lib.ptr(v[1]), _lib.ptr(v[2]), _lib.ptr(v[3]), _lib.ptr(v[4]), _lib.ptr(v[5]),
                                                 _lib.ptr(v[6]), _lib.ptr(v[7]), _lib.ptr(h), _lib.ptr(c), _lib.stream_ptr()))
    return h, c


def dcrnn_weight_image(wz, wr, wh, bz, br, bh, cin: int, K: int) -> Optional[torch.Tensor]:
    """B-operand image of the wgmma kernel for DConv weights (None when the configuration has no tensor kernel)."""
    cout = wz.size(-1)
    if cout != 32 or K != 2 or not (1 <= cin <= 4):
        return None
    img = torch.empty(int(_lib.lib().stmp_gru_weight_image_bytes()), dtype=torch.uint8, device=wz.device)
    args = [_f32c(w.detach(), "weight") for w in (wz, wr, wh)]
    bs = [None if b is None else _f32c(b.detach(), "bias") for b in (bz, br, bh)]
    with torch.cuda.device(wz.device):
        _lib.check(_lib.lib().stmp_dcrnn_pack_weights(cin, cout, K, _lib.ptr(args[0]), _lib.ptr(args[1]), _lib.ptr(args[2]),
                                                      _lib.ptr(bs[0]), _lib.ptr(bs[1]), _lib.ptr(bs[2]), _lib.ptr(img), _lib.stream_ptr()))
    return img


def gru_weight_image(wcat: torch.Tensor, bcat: torch.Tensor) -> torch.Tensor:
    img = torch.empty(int(_lib.lib().stmp_gru_weight_image_bytes()), dtype=torch.uint8, device=wcat.device)
    with torch.cuda.device(wcat.device):
        _lib.check(_lib.lib().stmp_gru_pack_weights(_lib.ptr(_f32c(wcat, "wcat")), _lib.ptr(_f32c(bcat, "bcat")), _lib.ptr(img),
                                                    _lib.stream_ptr()))
    return img


class PackCache(object):
    """Caches the packed (wcat, bcat) of a module until one of its parameters changes (host-side `_version`
    check, no device sync), so inference pays the packing once."""

    def __init__(self):
        self._key, self._val = None, None

    def get(self, params, build):
        key = tuple((p.data_ptr(), p._version) for p in params)
        if key != self._key:
            with torch.no_grad():
                self._val = build()
            self._key = key
        return self._val


def gru_zr(pz, pr, h):
    _require_numel("gru_zr", pz.numel(), pr=pr, h=h)
    pz, pr, h =_f32c(pz, "pz"), _f32c(pr, "pr"), _f32c(h, "h")
    z, r, hr = torch.empty_like(pz), torch.empty_like(pz), torch.empty_like(pz)
    with torch.cuda.device(pz.device):
        _lib.check(_lib.lib().stmp_gru_zr(pz.numel(), _lib.ptr(pz), _lib.ptr(pr), _lib.ptr(h), _lib.ptr(z), _lib.ptr(r),
                                          _lib.ptr(hr), _lib.stream_ptr()))
    return z, r, hr


def gru_out(ph, z, h):
    _require_numel("gru_out", ph.numel(), z=z, h=h)
    ph, z, h =_f32c(ph, "ph"), _f32c(z, "z"), _f32c(h, "h")
    hn = torch.empty_like(ph)
    with torch.cuda.device(ph.device):
        _lib.check(_lib.lib().stmp_gru_out(ph.numel(), _lib.ptr(ph), _lib.ptr(z), _lib.ptr(h), None, _lib.ptr(hn),
                                           _lib.stream_ptr()))
    return hn


def dcrnn_bwd_supported(plan: GraphPlan, cin: int, cout: int, K: int) -> bool:
    return bool(_lib.lib().stmp_dcrnn_bwd_supported(plan.handle, cin, cout, K))


def dcrnn_bwd_basis(plan: GraphPlan, x, out, h0, stash, S1, S2):
    """S1/S2 (T*B, N, ld) <- bases of [X_t | H_{t-1}] and [X_t | H_{t-1}*R_t] for every (t, b): one launch."""
    x, out, stash = _f32c(x, "x"), _f32c(out, "out"), _f32c(stash, "stash")
    B, T, N, Ci = x.shape
    h0 = None if h0 is None else _f32c(h0, "h0")
    with torch.cuda.device(x.device):
        _lib.check(_lib.lib().stmp_dcrnn_bwd_basis(plan.handle, B, T, Ci, out.size(-1), _lib.ptr(x), T * N * Ci, N * Ci, _lib.ptr(out),
                                                   _lib.ptr(h0), _lib.ptr(stash), _lib.ptr(S1), _lib.ptr(S2), S1.size(-1), _lib.stream_ptr()))


def dcrnn_bwd_seq(plan: GraphPlan, cin: int, gout, out, h0, stash, whsT, wzrT, dph_all, dpzr_all, dx, dh0):
    """The reverse-time recurrence of the DCRNN backward in one persistent launch (one CTA per window)."""
    gout, out, stash = _f32c(gout, "gout"), _f32c(out, "out"), _f32c(stash, "stash")
    B, T, N, Co = gout.shape
    h0 = None if h0 is None else _f32c(h0, "h0")
    with torch.cuda.device(gout.device):
        _lib.check(_lib.lib().stmp_dcrnn_bwd_seq(plan.handle, B, T, cin, Co, _lib.ptr(gout), _lib.ptr(out), _lib.ptr(h0), _lib.ptr(stash),
                                                 _lib.ptr(_f32c(whsT, "whsT")), _lib.ptr(_f32c(wzrT, "wzrT")), _lib.ptr(dph_all),
                                                 _lib.ptr(dpzr_all), _lib.ptr(dx), _lib.ptr(dh0), _lib.stream_ptr()))


def dcrnn_narrow_bwd_supported(plan: GraphPlan, cin: int, cout: int, K: int) -> bool:
    return bool(_lib.lib().stmp_dcrnn_narrow_bwd_supported(plan.handle, cin, cout, K))


def dcrnn_narrow_bwd_seq(plan: GraphPlan, cin: int, K: int, gout, out, h0, stash, whsT, wzrT, dph_all, dpzr_all, dx, dh0):
    """The reverse-time recurrence of the narrow-state DCRNN backward (cout <= 4, any K <= 4) in one persistent launch."""
    gout, out, stash = _f32c(gout, "gout"), _f32c(out, "out"), _f32c(stash, "stash")
    B, T, N, Co = gout.shape
    h0 = None if h0 is None else _f32c(h0, "h0")
    with torch.cuda.device(gout.device):
        _lib.check(_lib.lib().stmp_dcrnn_narrow_bwd_seq(plan.handle, B, T, cin, Co, K, _lib.ptr(gout), _lib.ptr(out), _lib.ptr(h0),
                                                        _lib.ptr(stash), _lib.ptr(_f32c(whsT, "whsT")), _lib.ptr(_f32c(wzrT, "wzrT")),
                                                        _lib.ptr(dph_all), _lib.ptr(dpzr_all), _lib.ptr(dx), _lib.ptr(dh0),
                                                        _lib.stream_ptr()))


def dcrnn_bwd_basis_ld(cin: int, cout: int, K: int) -> int:
    """Row pitch of the stacked bases: (2K-1)(cin+cout) rounded up to 8 floats (16-byte rows for the weight-gradient kernel's tiles)."""
    return ((2 * K - 1) * (cin + cout) + 7) // 8 * 8


def dcrnn_bwd_wgrad(cin: int, K: int, S1, S2, dpzr_all, dph_all, has_bias: bool):
    """(gz, gr, gh, gbz, gbr, gbh): weight / bias gradients of the three gates over all (t, b, n) rows in two launches
    (`stmp_dcrnn_bwd_wgrad`); S1 / S2 (T*B, N, ld) from dcrnn_bwd_basis with ld = dcrnn_bwd_basis_ld(...)."""
    Co = dph_all.size(-1)
    C = cin + Co
    dev = S1.device
    rows = S1.size(0) * S1.size(1)
    ws = _wgrad_workspace(dev, _lib.lib().stmp_dcrnn_bwd_wgrad_workspace_bytes, cin)
    g = torch.empty(3, 2, K, C, Co, device=dev, dtype=torch.float32)
    gb = torch.empty(3, Co, device=dev, dtype=torch.float32) if has_bias else None
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().stmp_dcrnn_bwd_wgrad(cin, Co, K, rows, S1.size(-1), _lib.ptr(S1), _lib.ptr(S2), _lib.ptr(dpzr_all), _lib.ptr(dph_all),
                                                   _lib.ptr(ws), _lib.ptr(g[0]), _lib.ptr(g[1]), _lib.ptr(g[2]),
                                                   _lib.ptr(None if gb is None else gb[0]), _lib.ptr(None if gb is None else gb[1]),
                                                   _lib.ptr(None if gb is None else gb[2]), _lib.stream_ptr()))
    if gb is None:
        return g[0], g[1], g[2], None, None, None
    return g[0], g[1], g[2], gb[0], gb[1], gb[2]


def adam_flat(param, grad, exp_avg, exp_avg_sq, step, ticket, lr, beta1, beta2, eps, weight_decay=0.0, grad_scale=1.0, zero_grad=True):
    """One-launch Adam over flat fp32 buffers (`stmp_adam_flat`); `step` (1 float) and `ticket` (1 int32, zero) are device tensors."""
    for t, nm in ((param, "param"), (grad, "grad"), (exp_avg, "exp_avg"), (exp_avg_sq, "exp_avg_sq")):
        if not (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() and t.numel() == param.numel()):
            raise RuntimeError(f"adam_flat: {nm} must be a contiguous CUDA fp32 buffer of {param.numel()} elements")
    with torch.cuda.device(param.device):
        _lib.check(_lib.lib().stmp_adam_flat(param.numel(), _lib.ptr(param), _lib.ptr(grad), _lib.ptr(exp_avg), _lib.ptr(exp_avg_sq), _lib.ptr(step),
                                             _lib.ptr(ticket), lr, beta1, beta2, eps, weight_decay, grad_scale, 1 if zero_grad else 0,
                                             _lib.stream_ptr()))


def dcrnn_pack_bwd_weights(wz, wr, wh, cin: int, K: int):
    """(whsT (Co, (2K-1)C), wzrT (2Co, (2K-1)C)): transposed stacked weights of the backward GEMMs, one launch."""
    Co = wz.size(-1)
    nbC = (2 * K - 1) * (cin + Co)
    whsT = torch.empty(Co, nbC, device=wz.device, dtype=torch.float32)
    wzrT = torch.empty(2 * Co, nbC, device=wz.device, dtype=torch.float32)
    with torch.cuda.device(wz.device):
        _lib.check(_lib.lib().stmp_dcrnn_pack_bwd_weights(cin, Co, K, _lib.ptr(_f32c(wz.detach(), "wz")), _lib.ptr(_f32c(wr.detach(), "wr")),
                                                          _lib.ptr(_f32c(wh.detach(), "wh")), _lib.ptr(whsT), _lib.ptr(wzrT), _lib.stream_ptr()))
    return whsT, wzrT


def _rows_entry(cin: int, cout: int, K: int) -> Optional[str]:
    """Prefix of the row-split library entries that serve (cin, cout, K), from the attributes alone; None outside every envelope."""
    if not 1 <= cin <= 4:
        return None
    if cout == 32 and K == 2:
        return "stmp_dcrnn_rows"
    if 1 <= cout <= 4 and 1 <= K <= 4:
        return "stmp_dcrnn_narrow_rows"
    if cout == 64 and K in (2, 3):
        return "stmp_dcrnn_wide_rows"
    return None


def dcrnn_rows_supported(plan: GraphPlan, cin: int, cout: int, K: int) -> bool:
    """The row-split DCRNN envelopes on a DConv plan, any graph size, cin 1..4: cout = 32 at K = 2 (stmp_dcrnn_rows_*), cout and K in
    1..4 (stmp_dcrnn_narrow_rows_*), cout = 64 at K = 2 or 3 (stmp_dcrnn_wide_rows_*).  The plan is consulted only inside an envelope."""
    entry = _rows_entry(cin, cout, K)
    return entry is not None and bool(getattr(_lib.lib(), entry + "_supported")(plan.handle, cin, cout, K))


def dcrnn_narrow_rows_supported(plan: GraphPlan, cin: int, cout: int, K: int) -> bool:
    """dcrnn_rows_supported restricted to the narrow row-split kernels (cout 1..4)."""
    return 1 <= cout <= 4 and dcrnn_rows_supported(plan, cin, cout, K)


def dcrnn_wide_rows_supported(plan: GraphPlan, cin: int, cout: int, K: int) -> bool:
    """dcrnn_rows_supported restricted to the 64-wide row-split kernels (cout = 64)."""
    return cout == 64 and dcrnn_rows_supported(plan, cin, cout, K)


def dcrnn_rows_fwd(plan: GraphPlan, x: torch.Tensor, wzrT: torch.Tensor, whsT: torch.Tensor, bz, br, bh,
                   win_start: Optional[torch.Tensor] = None, horizon: Optional[int] = None, train: bool = False):
    """Row-split BatchedDCRNN recurrence from H_0 = 0 (stmp_dcrnn_rows_fwd).  x: (B,T,N,cin) windows, or -- with win_start (int64 [B]) and
    horizon -- the resident series (T_total,N,cin) read in place.  wzrT / whsT from dcrnn_pack_bwd_weights; biases (32,) or None.
    Returns out (B,T,N,32); with `train`, (out, stash (T,B,N,96), S1, S2 (T*B, N, ld)) -- the operands of dcrnn_rows_bwd / dcrnn_bwd_wgrad."""
    x = _f32c(x, "X")
    N = plan.num_nodes
    if win_start is None:
        if x.dim() != 4 or x.size(2) != N:
            raise RuntimeError(f"X must be (B,T,{N},Cin), got {tuple(x.shape)}")
        B, T, _, cin = x.shape
        bstride, tstride, ws = T * N * cin, N * cin, None
    else:
        if x.dim() != 3 or x.size(1) != N:
            raise RuntimeError(f"series must be (T_total,{N},Cin), got {tuple(x.shape)}")
        _require_cuda(win_start, "win_start")
        ws = win_start.to(torch.int64).contiguous()
        B, T, cin = ws.numel(), int(horizon), x.size(2)
        bstride, tstride = 0, N * cin
    nb = 3 * (cin + 32)
    if wzrT.shape != (64, nb) or whsT.shape != (32, nb):
        raise RuntimeError(f"dcrnn_rows_fwd: wzrT must be (64, {nb}) and whsT (32, {nb})")
    f32 = dict(device=x.device, dtype=torch.float32)
    ld = dcrnn_bwd_basis_ld(cin, 32, 2)
    out = torch.empty(B, T, N, 32, **f32)
    st = S1 = S2 = None
    if train:
        st = torch.empty(T, B, N, 96, **f32)
        S1 = torch.empty(T * B, N, ld, **f32)
        S2 = torch.empty(T * B, N, ld, **f32)
    if B > 0 and T > 0:
        scr = torch.empty(int(_lib.lib().stmp_dcrnn_rows_scratch_bytes(plan.handle, B)) // 4, **f32)
        bs = [None if b is None else _f32c(b.detach(), "bias") for b in (bz, br, bh)]
        with torch.cuda.device(x.device):
            _lib.check(_lib.lib().stmp_dcrnn_rows_fwd(plan.handle, B, T, cin, _lib.ptr(x), _lib.ptr(ws), bstride, tstride,
                                                      _lib.ptr(_f32c(wzrT, "wzrT")), _lib.ptr(_f32c(whsT, "whsT")), _lib.ptr(bs[0]),
                                                      _lib.ptr(bs[1]), _lib.ptr(bs[2]), _lib.ptr(scr), _lib.ptr(out), _lib.ptr(st),
                                                      _lib.ptr(S1), _lib.ptr(S2), ld, _lib.stream_ptr()))
    return (out, st, S1, S2) if train else out


def dcrnn_rows_bwd(plan: GraphPlan, cin: int, gout, out, stash, wzrT, whsT, want_dx: bool):
    """(dph_all (T,B,N,32), dpzr_all (T,B,N,64), dx (B,T,N,cin) or None): the reverse-time backward of dcrnn_rows_fwd (stmp_dcrnn_rows_bwd)."""
    gout = _f32c(gout, "gout")
    B, T, N, _ = gout.shape
    f32 = dict(device=gout.device, dtype=torch.float32)
    dph, dpzr = torch.empty(T, B, N, 32, **f32), torch.empty(T, B, N, 64, **f32)
    dx = torch.empty(B, T, N, cin, **f32) if want_dx else None
    if B > 0 and T > 0:
        scr = torch.empty(int(_lib.lib().stmp_dcrnn_rows_scratch_bytes(plan.handle, B)) // 4, **f32)
        with torch.cuda.device(gout.device):
            _lib.check(_lib.lib().stmp_dcrnn_rows_bwd(plan.handle, B, T, cin, _lib.ptr(gout), _lib.ptr(out), _lib.ptr(stash), _lib.ptr(wzrT),
                                                      _lib.ptr(whsT), _lib.ptr(scr), _lib.ptr(dph), _lib.ptr(dpzr), _lib.ptr(dx),
                                                      _lib.stream_ptr()))
    return dph, dpzr, dx


def _x_blocks(plan: GraphPlan, buf: torch.Tensor, width: int, pitch: int, K: int, cols=spmm_cols):
    """In place in buf (rows, N, LD) holding U in columns [0, width): the diffusion blocks [U | P_o U | P_i U | 2 P_o T_1o - U | ...],
    block j at column j * pitch (2(K-1) launches of stmp_spmm over all rows).  `cols` is the column-block product, `spmm_cols`; the
    DCRNN backward passes the one of the `ops` it runs against."""
    for k in range(1, K):
        for o in (0, 1):
            dst = (1 + 2 * (k - 1) + o) * pitch
            if k == 1:
                cols(plan, o, buf, 0, dst, width)
            else:
                cols(plan, o, buf, dst - 2 * pitch, dst, width, alpha=2.0, z_col=0, beta=-1.0)


def _x_blocks_adjoint(plan: GraphPlan, buf: torch.Tensor, width: int, pitch: int, K: int, cols=spmm_cols):
    """In place: columns [0, width) of buf (rows, N, LD) <- the transposed adjoint of U -> _x_blocks(U) applied to the blocks of buf."""
    for k in range(K - 1, 1, -1):                                                  # T_k = 2 P T_{k-1} - U
        for o in (0, 1):
            src = (1 + 2 * (k - 1) + o) * pitch
            cols(plan, o, buf, src, src - 2 * pitch, width, alpha=2.0, z_col=src - 2 * pitch, beta=1.0, transposed=True)
            buf[..., :width].sub_(buf[..., src:src + width])
    if K > 1:                                                                      # T_1 = P U
        cols(plan, 0, buf, pitch, 0, width, z_col=0, beta=1.0, transposed=True)
        cols(plan, 1, buf, 2 * pitch, 0, width, z_col=0, beta=1.0, transposed=True)


def _hoisted_entry(cout: int, what: str):
    """stmp_dcrnn_wide_rows_<what> at 64 hidden channels, stmp_dcrnn_narrow_rows_<what> otherwise (its checks refuse all but cout 1..4);
    the two families take the same arguments."""
    return getattr(_lib.lib(), ("stmp_dcrnn_wide_rows_" if cout == 64 else "stmp_dcrnn_narrow_rows_") + what)


def _hoisted_scratch(plan: GraphPlan, B: int, cout: int, K: int, device) -> Optional[torch.Tensor]:
    nbytes = int(_hoisted_entry(cout, "scratch_bytes")(plan.handle, B, cout, K))
    return torch.empty(nbytes // 4, device=device, dtype=torch.float32) if nbytes else None


_NROWS_XBUF_BYTES = 256 << 20      # inference: windows are chunked so that the hoisted X blocks stay under this size


def dcrnn_hoisted_rows_fwd(plan: GraphPlan, x: torch.Tensor, wzrT: torch.Tensor, whsT: torch.Tensor, bz, br, bh, K: int,
                           win_start: Optional[torch.Tensor] = None, horizon: Optional[int] = None, train: bool = False):
    """Row-split BatchedDCRNN recurrence from H_0 = 0 with the X diffusion hoisted out of the time loop: stmp_dcrnn_narrow_rows_fwd for
    cout 1..4, stmp_dcrnn_wide_rows_fwd for cout = 64 (cout = whsT.size(0)).  x: (B,T,N,cin) windows, or -- with win_start (int64 [B]) and
    horizon, inference only -- the resident series (T_total,N,cin), whose windows are gathered into the hoisted X blocks.  wzrT / whsT from
    dcrnn_pack_bwd_weights; biases (cout,) or None.  Returns out (B,T,N,cout); with `train`, (out, stash, S1, S2 (T*B, N, (2K-1)C)) -- the
    operands of dcrnn_hoisted_rows_bwd and of the weight gradients."""
    x = _f32c(x, "X")
    N = plan.num_nodes
    if win_start is None:
        if x.dim() != 4 or x.size(2) != N:
            raise RuntimeError(f"X must be (B,T,{N},Cin), got {tuple(x.shape)}")
        B, T, _, cin = x.shape
    else:
        if train:
            raise RuntimeError("dcrnn_hoisted_rows_fwd: win_start is an inference entry")
        if x.dim() != 3 or x.size(1) != N:
            raise RuntimeError(f"series must be (T_total,{N},Cin), got {tuple(x.shape)}")
        _require_cuda(win_start, "win_start")
        win_start = win_start.to(torch.int64).contiguous()
        B, T, cin = win_start.numel(), int(horizon), x.size(2)
    cout = whsT.size(0)
    C = cin + cout
    nbc = (2 * K - 1) * C
    if wzrT.shape != (2 * cout, nbc) or whsT.shape != (cout, nbc):
        raise RuntimeError(f"dcrnn_hoisted_rows_fwd: wzrT must be ({2 * cout}, {nbc}) and whsT ({cout}, {nbc})")
    f32 = dict(device=x.device, dtype=torch.float32)
    wzrT, whsT = _f32c(wzrT, "wzrT"), _f32c(whsT, "whsT")
    bs = [None if b is None else _f32c(b.detach(), "bias") for b in (bz, br, bh)]
    out = torch.empty(B, T, N, cout, **f32)
    fwd = _hoisted_entry(cout, "fwd")

    def run(Bc, xp, strides, o, st, S1, S2, scr):
        with torch.cuda.device(x.device):
            _lib.check(fwd(plan.handle, Bc, T, cin, cout, K, _lib.ptr(xp), *strides, _lib.ptr(wzrT), _lib.ptr(whsT), _lib.ptr(bs[0]),
                           _lib.ptr(bs[1]), _lib.ptr(bs[2]), _lib.ptr(scr), _lib.ptr(o), _lib.ptr(st), _lib.ptr(S1), _lib.ptr(S2),
                           _lib.stream_ptr()))

    if train:
        if cout == 64:
            st = torch.empty(T, B, N, 192, **f32)
        else:                               # node-major, the windows along the lanes; cout padded to 1, 2 or 4 floats
            st = torch.empty(T, N, B, 3 * (4 if cout == 3 else cout), **f32)
        S1 = torch.empty(T * B, N, nbc, **f32)
        S2 = torch.empty(T * B, N, nbc, **f32)
        if B > 0 and T > 0:
            S1.view(T, B, N, nbc)[..., :cin] = x.transpose(0, 1)
            _x_blocks(plan, S1, cin, C, K)
            run(B, None, (0, 0, 0, 0), out, st, S1, S2, _hoisted_scratch(plan, B, cout, K, x.device))
        return out, st, S1, S2
    if B == 0 or T == 0:
        return out
    if K == 1:                                  # the X "blocks" are X itself, read in place
        if win_start is not None:
            x = window_gather(x, win_start, T, with_target=False)
        run(B, x, (T * N * cin, N * cin, cin, cin), out, None, None, None, _hoisted_scratch(plan, B, cout, K, x.device))
        return out
    w = (2 * K - 1) * cin
    Bc = max(1, min(B, _NROWS_XBUF_BYTES // (T * N * w * 4)))
    scr = _hoisted_scratch(plan, Bc, cout, K, x.device)
    buf = torch.empty(Bc * T, N, w, **f32)
    for b0 in range(0, B, Bc):
        nb = min(Bc, B - b0)
        xb = buf[:nb * T]
        if win_start is None:
            xb.view(nb, T, N, w)[..., :cin] = x[b0:b0 + nb]
        else:
            xb.view(nb, T, N, w)[..., :cin] = window_gather(x, win_start[b0:b0 + nb], T, with_target=False)
        _x_blocks(plan, xb, cin, cin, K)
        run(nb, xb, (T * N * w, N * w, w, cin), out[b0:b0 + nb], None, None, None, scr)
    return out


def dcrnn_hoisted_rows_bwd(plan: GraphPlan, cin: int, K: int, gout, out, stash, wzrT, whsT, want_dx: bool):
    """(dph_all (T,B,N,cout), dpzr_all (T,B,N,2cout), dx (B,T,N,cin) or None): the reverse-time backward of dcrnn_hoisted_rows_fwd
    (stmp_dcrnn_narrow_rows_bwd or stmp_dcrnn_wide_rows_bwd), then dX from the X columns of dS1 + dS2 through one hoisted transposed
    basis adjoint."""
    gout = _f32c(gout, "gout")
    B, T, N, cout = gout.shape
    f32 = dict(device=gout.device, dtype=torch.float32)
    dph, dpzr = torch.empty(T, B, N, cout, **f32), torch.empty(T, B, N, 2 * cout, **f32)
    w = (2 * K - 1) * cin
    dsx = torch.empty(T * B, N, w, **f32) if want_dx else None
    if B > 0 and T > 0:
        scr = _hoisted_scratch(plan, B, cout, K, gout.device)
        with torch.cuda.device(gout.device):
            _lib.check(_hoisted_entry(cout, "bwd")(plan.handle, B, T, cin, cout, K, _lib.ptr(gout), _lib.ptr(out), _lib.ptr(stash),
                                                   _lib.ptr(wzrT), _lib.ptr(whsT), _lib.ptr(scr), _lib.ptr(dph), _lib.ptr(dpzr),
                                                   _lib.ptr(dsx), w, _lib.stream_ptr()))
    if not want_dx:
        return dph, dpzr, None
    if B == 0 or T == 0:
        return dph, dpzr, torch.zeros(B, T, N, cin, **f32)
    _x_blocks_adjoint(plan, dsx, cin, cin, K)
    return dph, dpzr, dsx.view(T, B, N, w)[..., :cin].transpose(0, 1).contiguous()


class _MaskedMAE(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pred, target):
        pred, target = _f32c(pred, "pred"), _f32c(target, "target")
        if pred.shape != target.shape:
            raise RuntimeError(f"masked_mae: shape mismatch {tuple(pred.shape)} vs {tuple(target.shape)}")
        ws = torch.empty(int(_lib.lib().stmp_masked_mae_workspace_floats()), device=pred.device, dtype=torch.float32)
        out = torch.empty(2, device=pred.device, dtype=torch.float32)           # [loss, sum(mask)]
        with torch.cuda.device(pred.device):
            _lib.check(_lib.lib().stmp_masked_mae_fwd(pred.numel(), _lib.ptr(pred), _lib.ptr(target), _lib.ptr(ws), ctypes.c_void_p(out.data_ptr()),
                                                      ctypes.c_void_p(out.data_ptr() + 4), _lib.stream_ptr()))
        ctx.save_for_backward(pred, target, out)
        return out[0].clone()

    @staticmethod
    def backward(ctx, gout):
        pred, target, out = ctx.saved_tensors
        gp = torch.empty_like(pred)
        gout = gout.contiguous().to(torch.float32)
        with torch.cuda.device(pred.device):
            _lib.check(_lib.lib().stmp_masked_mae_bwd(pred.numel(), _lib.ptr(pred), _lib.ptr(target), ctypes.c_void_p(out.data_ptr() + 4),
                                                      _lib.ptr(gout), _lib.ptr(gp), _lib.stream_ptr()))
        return gp, None


def masked_mae(pred: torch.Tensor, target: torch.Tensor) -> torch.Tensor:
    """Fused masked MAE (forward 2 launches, backward 1) with the semantics of examples/indexBatching/DCRNN/utils.py:10-18."""
    return _MaskedMAE.apply(pred, target)


def _slice_ptr(t: Optional[torch.Tensor]):
    """(pointer, batch stride in elements) of a (B, N, C) fp32 slice whose trailing two dims are dense."""
    if t is None:
        return None, 0
    if t.dtype != torch.float32 or t.dim() != 3 or t.stride(2) != 1 or t.stride(1) != t.size(2):
        raise RuntimeError("expected a float32 (B, N, C) slice with dense trailing dims")
    return ctypes.c_void_p(t.data_ptr()), t.stride(0)


def gru_bwd_carry(cin: int, cout: int, du2, du1, g_prev=None, z_prev=None, r_prev=None, dx=None, gout=None, z=None, ht=None,
                  g=None, dph=None, dh_out=None):
    """stmp_gru_bwd_carry: close step t+1 (g_prev, z_prev, r_prev, du2, du1 [, dx]) and/or open step t (gout, z, ht -> g, dph)."""
    ref = g_prev if g_prev is not None else gout
    B, N = ref.size(0), ref.size(1)
    du_ld = du2.size(-1)
    zp, s1 = _slice_ptr(z_prev)
    rp, _ = _slice_ptr(r_prev)
    zz, s2 = _slice_ptr(z)
    hh, _ = _slice_ptr(ht)
    go, gs = _slice_ptr(gout)
    dxp, dxs = _slice_ptr(dx)
    stash_bs = s1 if z_prev is not None else s2
    if z_prev is not None and z is not None and s1 != s2:
        raise RuntimeError("stash slices of one call must share their batch stride")
    with torch.cuda.device(ref.device):
        _lib.check(_lib.lib().stmp_gru_bwd_carry(B, N, cin, cout, du_ld, _lib.ptr(g_prev), zp, rp, _lib.ptr(du2), _lib.ptr(du1), dxp, dxs,
                                                 go, gs, zz, hh, stash_bs, _lib.ptr(g), _lib.ptr(dph), _lib.ptr(dh_out), _lib.stream_ptr()))


def gru_bwd_zr(cin: int, cout: int, g, hprev, z, r, ht, du2, dpzr):
    B, N = g.size(0), g.size(1)
    hp, hs = _slice_ptr(hprev)
    zz, ss = _slice_ptr(z)
    rr, _ = _slice_ptr(r)
    hh, _ = _slice_ptr(ht)
    with torch.cuda.device(g.device):
        _lib.check(_lib.lib().stmp_gru_bwd_zr(B, N, cin, cout, du2.size(-1), _lib.ptr(g), hp, hs, zz, rr, hh, ss, _lib.ptr(du2),
                                              _lib.ptr(dpzr), _lib.stream_ptr()))


def lstm_ifc(pi, pf, pc, c, wci, wcf, bi, bf, bc):
    cout = pi.size(-1)
    rows = pi.numel() // cout
    _require_numel("lstm_ifc", rows * cout, pf=pf, pc=pc, c=c)
    _require_numel("lstm_ifc", cout, wci=wci, wcf=wcf, bi=bi, bf=bf, bc=bc)
    pi, pf, pc, c = (_f32c(t, "gate") for t in (pi, pf, pc, c))
    cn = torch.empty_like(pi)
    v = [_f32c(t.detach().reshape(-1), "param") for t in (wci, wcf, bi, bf, bc)]
    with torch.cuda.device(pi.device):
        _lib.check(_lib.lib().stmp_lstm_ifc(rows, cout, _lib.ptr(pi), _lib.ptr(pf), _lib.ptr(pc), _lib.ptr(c), _lib.ptr(v[0]),
                                            _lib.ptr(v[1]), _lib.ptr(v[2]), _lib.ptr(v[3]), _lib.ptr(v[4]), None, None, None,
                                            _lib.ptr(cn), _lib.stream_ptr()))
    return cn


def lstm_oh(po, cnew, wco, bo):
    cout = po.size(-1)
    rows = po.numel() // cout
    _require_numel("lstm_oh", rows * cout, cnew=cnew)
    _require_numel("lstm_oh", cout, wco=wco, bo=bo)
    po, cnew = _f32c(po, "po"), _f32c(cnew, "cnew")
    hn = torch.empty_like(po)
    v = [_f32c(t.detach().reshape(-1), "param") for t in (wco, bo)]
    with torch.cuda.device(po.device):
        _lib.check(_lib.lib().stmp_lstm_oh(rows, cout, _lib.ptr(po), _lib.ptr(cnew), _lib.ptr(v[0]), _lib.ptr(v[1]), None,
                                           _lib.ptr(hn), _lib.stream_ptr()))
    return hn


def lstm_gate_bwd(pre, c_old, c_new, gh, gc, wci, wcf, wco, bi, bf, bc, bo):
    """(dpre (rows,4Co), dC_old (rows,Co)) of the peephole-LSTM gate chain (stmp_lstm_gate_bwd); gh / gc may be None."""
    cout = c_old.size(-1)
    rows = c_old.numel() // cout
    _require_numel("lstm_gate_bwd", rows * 4 * cout, pre=pre)
    _require_numel("lstm_gate_bwd", rows * cout, c_new=c_new, gh=gh, gc=gc)
    _require_numel("lstm_gate_bwd", cout, wci=wci, wcf=wcf, wco=wco, bi=bi, bf=bf, bc=bc, bo=bo)
    pre, c_old, c_new = _f32c(pre, "pre"), _f32c(c_old, "c_old"), _f32c(c_new, "c_new")
    dpre = torch.empty_like(pre)
    dco = torch.empty_like(c_old)
    gh = None if gh is None else _f32c(gh, "gh")
    gc = None if gc is None else _f32c(gc, "gc")
    v = [_f32c(t.detach().reshape(-1), "param") for t in (wci, wcf, wco, bi, bf, bc, bo)]
    with torch.cuda.device(pre.device):
        _lib.check(_lib.lib().stmp_lstm_gate_bwd(rows, cout, _lib.ptr(pre), _lib.ptr(c_old), _lib.ptr(c_new), _lib.ptr(gh), _lib.ptr(gc),
                                                 *[_lib.ptr(t) for t in v], _lib.ptr(dpre), _lib.ptr(dco), _lib.stream_ptr()))
    return dpre, dco


def window_gather(series: torch.Tensor, start: torch.Tensor, horizon: int, with_target: bool = True):
    """x[b] = series[start[b]:start[b]+h], y[b] = series[start[b]+h:start[b]+2h] (index_dataset.py:49-57)."""
    series = _f32c(series, "series")
    _require_cuda(start, "start")
    start = start.to(torch.int64).contiguous()
    B = start.numel()
    row = series[0].numel()
    shape = (B, horizon) + tuple(series.shape[1:])
    x = torch.empty(shape, dtype=torch.float32, device=series.device)
    y = torch.empty(shape, dtype=torch.float32, device=series.device) if with_target else None
    with torch.cuda.device(series.device):
        _lib.check(_lib.lib().stmp_window_gather(_lib.ptr(series), series.size(0), row, _lib.ptr(start), B, horizon,
                                                 _lib.ptr(x), _lib.ptr(y), _lib.stream_ptr()))
    return (x, y) if with_target else x


def hetero_lstm_supported(out_channels: int, in_channels: int, num_rel: int) -> bool:
    return bool(_lib.lib().stmp_hetero_lstm_supported(out_channels, in_channels, num_rel))


def _hetero_desc(types):
    """stmp_hetero_lstm_fwd / _bwd's desc of `types` (see hetero_lstm_fwd) and the contiguous float32 operands it points at."""
    desc = (ctypes.c_int64 * (_lib.HETERO_DESC * len(types)))()
    ops_ = []
    for t, (x, h, c, w, b, plans, sources, src_idx, ranks) in enumerate(types):
        x, w, b = _f32c(x.detach(), "X"), _f32c(w, "w"), _f32c(b, "b")
        h = None if h is None else _f32c(h.detach(), "H")
        c = None if c is None else _f32c(c.detach(), "C")
        srcs = [None if s is None else _f32c(s.detach(), "H") for s in sources]
        R, pad = len(plans), [0] * (_lib.HETERO_MAX_REL - len(plans))
        row = [x.size(0), x.size(1), R] + [_addr(v) for v in (x, h, c, w, b)] + [0, 0]
        row += [p.handle.value for p in plans] + pad + [_addr(v) for v in srcs] + pad + [0] * (_lib.HETERO_DESC - 18)
        row[30:30 + R], row[34:34 + R] = list(src_idx), list(ranks)
        desc[t * _lib.HETERO_DESC:(t + 1) * _lib.HETERO_DESC] = row
        ops_.append(dict(x=x, h=h, c=c, w=w, srcs=srcs, n=x.size(0), cin=x.size(1), R=R))
    return desc, ops_


def _addr(v):
    return 0 if v is None else v.data_ptr()


def _set(desc, t, field, v):
    desc[t * _lib.HETERO_DESC + field] = _addr(v)


def hetero_lstm_fwd(out_channels: int, types, has_h: bool, train: bool = False):
    """One HeteroGCLSTM step for every destination type in one launch (stmp_hetero_lstm_fwd).  `types`: per type a tuple
    (x (N, in), h (N, out) or None, c (N, out) or None, w (4 out, nb), b (4 out), plans, sources, src_idx, ranks) with `plans` the
    BipartitePlans of its incoming edge types, `sources` their source states (N_s, out) (None without H), `src_idx` the position of each
    source type in `types` and `ranks` each edge type's position in the metadata (both read by the backward only).  Returns
    [(H', C')] in `types` order; with `train`, also (desc, operands) for hetero_lstm_bwd, the stash and basis rows included.  No
    autograd."""
    desc, ops_ = _hetero_desc(types)
    dev = types[0][0].device
    outs = []
    for t, o in enumerate(ops_):
        hout = torch.empty(o["n"], out_channels, device=dev, dtype=torch.float32)
        cout = torch.empty_like(hout)
        _set(desc, t, 8, hout)
        _set(desc, t, 9, cout)
        outs.append((hout, cout))
        o["cout"] = cout
        if train:
            o["stash"] = torch.empty(4, o["n"], out_channels, device=dev, dtype=torch.float32)
            o["S"] = torch.empty(o["n"], o["cin"] + out_channels * (1 + o["R"]), device=dev, dtype=torch.float32)
            _set(desc, t, 18, o["stash"])
            _set(desc, t, 19, o["S"])
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().stmp_hetero_lstm_fwd(out_channels, len(types), desc, int(has_h), _lib.stream_ptr()))
    return (outs, desc, ops_) if train else outs


def hetero_lstm_bwd(out_channels: int, desc, ops_, gh, gc, want_dx, want_dh: bool, want_dc, want_dw: bool):
    """The backward of a training hetero_lstm_fwd (stmp_hetero_lstm_bwd, at most four launches): gh / gc per type (None: zero), want_dx /
    want_dc per type.  Returns per type (dx, dh, dc, dw (4 out, nb), db (4 out)), each None when not asked for."""
    dev = ops_[0]["x"].device
    res, keep = [], []
    for t, o in enumerate(ops_):
        g = [None if v is None else _f32c(v, "grad") for v in (gh[t], gc[t])]
        new = lambda *shape: torch.empty(*shape, device=dev, dtype=torch.float32)
        n, R = o["n"], o["R"]
        nb = o["cin"] + out_channels * (1 + R)
        r = dict(dpre=new(n, 4 * out_channels), dx=new(n, o["cin"]) if want_dx[t] else None, dh=new(n, out_channels) if want_dh else None,
                 dc=new(n, out_channels) if want_dc[t] else None, q=[new(n, out_channels) for _ in range(R)] if want_dh else [],
                 dw=new(4 * out_channels, nb + 1) if want_dw else None)
        for f, v in ((20, g[0]), (21, g[1]), (22, r["dpre"]), (23, r["dx"]), (24, r["dh"]), (25, r["dc"]), (38, r["dw"])):
            _set(desc, t, f, v)
        for k, q in enumerate(r["q"]):
            _set(desc, t, 26 + k, q)
        keep += g
        res.append(r)
    L_ = _lib.lib()
    ws = torch.empty(int(L_.stmp_hetero_lstm_workspace_bytes(out_channels, len(ops_), desc)) if want_dw else 0, device=dev,
                     dtype=torch.uint8)
    with torch.cuda.device(dev):
        _lib.check(L_.stmp_hetero_lstm_bwd(out_channels, len(ops_), desc, int(want_dh), _lib.ptr(ws) if want_dw else None,
                                           _lib.stream_ptr()))
    out = []
    for o, r in zip(ops_, res):
        nb = r["dw"].size(1) - 1 if want_dw else 0
        out.append((r["dx"], r["dh"], r["dc"], r["dw"][:, :nb] if want_dw else None, r["dw"][:, nb] if want_dw else None))
    return out


class _HeteroLstmFn(torch.autograd.Function):
    """Training form of hetero_lstm_fwd for T node types.  forward = the inference launch with the stash and the basis rows (so H', C'
    are bit-identical to the no_grad call), kept in ctx with the desc; backward = hetero_lstm_bwd: dX, dH, dC where asked for, and each
    type's packed weight / bias gradient handed to `params` as blocks described by its spec (see _spec_grads).  Inputs: X (T), H (T),
    C (T), then every type's parameters; outputs: H' (T), C' (T)."""

    @staticmethod
    def forward(ctx, out_channels, layout, specs, *flat):
        ctx.set_materialize_grads(False)
        T = len(layout)
        xs, hs, cs, params = flat[:T], flat[T:2 * T], flat[2 * T:3 * T], flat[3 * T:]
        types = [(xs[t], hs[t], cs[t]) + tuple(layout[t]) for t in range(T)]
        outs, ctx.desc, ctx.ops = hetero_lstm_fwd(out_channels, types, hs[0] is not None, train=True)
        ctx.out, ctx.T, ctx.specs, ctx.shapes = out_channels, T, specs, [p.shape for p in params]
        ctx.has_h, ctx.has_c = hs[0] is not None, cs[0] is not None
        return (*[o[0] for o in outs], *[o[1] for o in outs])

    @staticmethod
    def backward(ctx, *grads):
        T, need = ctx.T, ctx.needs_input_grad
        if all(g is None for g in grads):
            return (None,) * len(need)
        want_dx = [need[3 + t] for t in range(T)]
        want_dh = ctx.has_h and any(need[3 + T + t] for t in range(T))
        want_dc = [ctx.has_c and need[3 + 2 * T + t] for t in range(T)]
        want_dw = any(need[3 + 3 * T:])
        res = hetero_lstm_bwd(ctx.out, ctx.desc, ctx.ops, grads[:T], grads[T:], want_dx, want_dh, want_dc, want_dw)
        pgrads = []
        for t, (dx, dh, dc, dw, db) in enumerate(res):
            if want_dw:
                pgrads += _spec_grads(ctx.specs[t], dw, db)
            else:
                pgrads += [None] * len(ctx.specs[t])
        pgrads = [None if g is None else g.reshape(s) for g, s in zip(pgrads, ctx.shapes)]
        return (None, None, None, *[r[0] for r in res], *[r[1] if want_dh else None for r in res],
                *[r[2] for r in res], *pgrads)


def hetero_lstm_train(out_channels: int, types, params, specs):
    """Differentiable hetero_lstm_fwd: `types` as there; `params` the flat list of every type's parameters and `specs` per type the
    packed blocks they receive.  Returns [(H', C')]."""
    layout = [tuple(t[3:]) for t in types]
    flat = [t[0] for t in types] + [t[1] for t in types] + [t[2] for t in types]
    outs = _HeteroLstmFn.apply(out_channels, layout, specs, *flat, *params)
    T = len(types)
    return [(outs[t], outs[T + t]) for t in range(T)]


def bipartite_mean(plan, edge_index: torch.Tensor, h_src: torch.Tensor) -> torch.Tensor:
    """SAGEConv's mean of the source rows h_src (N_src, F) onto the plan's N_dst destination rows (0 for a row without edges): float32
    through spmm on the BipartitePlan (autograd through its source CSR), other dtypes by index_add over edge_index."""
    if h_src.size(0) != plan.num_src:
        raise RuntimeError(f"source state has {h_src.size(0)} rows, the edge type's plan {plan.num_src}")
    if h_src.dtype == torch.float32:
        pad = plan.num_nodes - h_src.size(0)
        x = torch.cat([h_src, h_src.new_zeros(pad, h_src.size(1))]) if pad else h_src
        return spmm(plan, 0, x)[:plan.num_dst]
    src, dst = edge_index[0], edge_index[1]
    agg = h_src.new_zeros(plan.num_dst, h_src.size(1)).index_add(0, dst, h_src[src])
    cnt = torch.zeros(plan.num_dst, dtype=h_src.dtype, device=h_src.device).index_add_(0, dst, torch.ones_like(dst, dtype=h_src.dtype))
    return agg / cnt.clamp(min=1).unsqueeze(1)
