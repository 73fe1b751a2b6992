"""DCRNN family behind the reference's module surface (drop-in for
torch_geometric_temporal/nn/recurrent/dcrnn.py: DConv :7-111, DCRNN :114-219, BatchedDConv :222-325,
BatchedDCRNN :328-475).  Same constructor signatures, forward signatures and state_dict keys
(`conv_x_{z,r,h}.weight (2,K,Cin+Cout,Cout)`, `.bias (Cout)`); the arithmetic runs in libstmp:

* inference (no grad): the whole recurrence in ONE fused kernel (`stmp_dcrnn_seq_fwd`);
* graphs too large for one SM (hidden 32, K = 2, Cin <= 4): BatchedDCRNN runs the row-split kernels (`stmp_dcrnn_rows_*`), two
  launches per step for all windows, and a hand-written reverse-time backward (`_DcrnnRowsFn`);
* graphs too large for one SM at narrow states (cout, Cin, K <= 4: the reference's BatchedDCRNN(F, F, K=3)), and hidden 64 at K = 2, 3
  on any graph: BatchedDCRNN runs the narrow / 64-wide row-split kernels (`stmp_dcrnn_narrow_rows_*`, `stmp_dcrnn_wide_rows_*`),
  2(K-1) launches per step for all windows after one hoisted diffusion of X, and a hand-written reverse-time backward
  (`_DcrnnHoistedRowsFn`);
* training / shapes the fused kernels cannot take: the tiled path = hand-written SpMM (`stmp_spmm`,
  differentiable through its transposed product) + cuBLAS contraction, with the diffusion shared
  between the z and r gates.
"""
import torch

from ... import ops
from ... import _lib
from ...ops import _x_blocks, _x_blocks_adjoint
from ...plan import PlanCache, _require_cuda


def _basis(plan, U: torch.Tensor, K: int):
    """[U, P_o U, P_i U, 2 P_o T - U, ...] for U (N,C) or (B,N,C); T_k = 2 P T_{k-1} - U for every
    k >= 2 (the reference never advances Tx_0 past X, dcrnn.py:80,106)."""
    blocks = [U]
    To = Ti = None
    for k in range(1, K):
        if k == 1:
            To, Ti = ops.spmm(plan, 0, U), ops.spmm(plan, 1, U)
        else:
            To = ops.spmm(plan, 0, To, alpha=2.0, z=U, beta=-1.0)
            Ti = ops.spmm(plan, 1, Ti, alpha=2.0, z=U, beta=-1.0)
        blocks += [To, Ti]
    return blocks


def _stack_weight(weight: torch.Tensor) -> torch.Tensor:
    """(2,K,C,O) -> ((2K-1)*C, O) matching `_basis` block order; block 0 = W[0,0] + W[1,0]."""
    K = weight.size(1)
    parts = [weight[0, 0] + weight[1, 0]]
    for k in range(1, K):
        parts += [weight[0, k], weight[1, k]]
    return torch.cat(parts, dim=0)


_UNSTACK_INDEX = {}
_SIDE_STREAMS = {}


def _side_stream(device) -> "torch.cuda.Stream":
    key = torch.device(device).index
    if key not in _SIDE_STREAMS:
        _SIDE_STREAMS[key] = torch.cuda.Stream(device=device)
    return _SIDE_STREAMS[key]


def _unstack_weight_grad(dWs: torch.Tensor, K: int, C: int) -> torch.Tensor:
    """((2K-1)*C, O) gradient of `_stack_weight(W)` -> gradient of W (2,K,C,O): one gather of basis blocks
    (block 0 feeds both W[0,0] and W[1,0]; block 1+2(k-1)+o feeds W[o,k])."""
    key = (K, dWs.device)
    idx = _UNSTACK_INDEX.get(key)
    if idx is None:
        order = [0 if k == 0 else 1 + 2 * (k - 1) + o for o in (0, 1) for k in range(K)]
        idx = torch.tensor(order, dtype=torch.long, device=dWs.device)
        _UNSTACK_INDEX[key] = idx
    O = dWs.size(1)
    return dWs.reshape(2 * K - 1, C, O).index_select(0, idx).view(2, K, C, O)


def _weight_grads(S1, S2, dph_all, dpzr_all, K, C, Co, has_bias):
    """(gz, gr, gh, gbz, gbr, gbh): weight / bias gradients over all (t, b, n) rows.  A single (3C x rows) @ (rows x Co) GEMM has only a
    handful of output tiles (cuBLAS runs it on 2 CTAs); chunking the row axis gives every SM a partial product to reduce."""
    rows, nbC = S1.size(0) * S1.size(1), S1.size(-1)
    chunks = 1
    for c in (128, 96, 64, 48, 32, 16, 8, 4, 2):
        if rows % c == 0:
            chunks = c
            break
    per = rows // chunks
    dWh = torch.bmm(S2.view(chunks, per, nbC).transpose(1, 2), dph_all.view(chunks, per, Co)).sum(0)
    dWzr = torch.bmm(S1.view(chunks, per, nbC).transpose(1, 2), dpzr_all.view(chunks, per, 2 * Co)).sum(0)
    gz = _unstack_weight_grad(dWzr[:, :Co], K, C)
    gr = _unstack_weight_grad(dWzr[:, Co:], K, C)
    gh = _unstack_weight_grad(dWh, K, C)
    if not has_bias:
        return gz, gr, gh, None, None, None
    ones = S1.new_ones(chunks, 1, per)
    dbzr = torch.bmm(ones, dpzr_all.view(chunks, per, 2 * Co)).sum(dim=(0, 1))
    dbh = torch.bmm(ones, dph_all.view(chunks, per, Co)).sum(dim=(0, 1))
    return gz, gr, gh, dbzr[:Co], dbzr[Co:], dbh


def _rows_param_grads(ctx, S1, cout, grads):
    """The six weight / bias gradients of a row-split Function (inputs 1..6): None when no parameter needs one, zeros when there are no
    windows or no steps (nothing to contract), else `grads()`."""
    if not any(ctx.needs_input_grad[1:7]):
        return [None] * 6
    if S1.numel() == 0:
        z = torch.zeros(2, ctx.K, ctx.cin + cout, cout, device=S1.device)
        return [z, z.clone(), z.clone()] + ([torch.zeros(cout, device=S1.device) for _ in range(3)] if ctx.has_bias else [None] * 3)
    return list(grads())


class _DcrnnSeqFn(torch.autograd.Function):
    """Training path of the recurrence: forward = ONE fused launch that also stashes (Z, R, H~) per step; backward =
    hand-written reverse-time loop over the stash (transposed SpMM for the diffusion adjoints, cuBLAS for the
    contractions).  Replaces autograd's replay of the ~1500-launch tiled graph."""

    fused_backward = True    # False forces the per-step backward even where a persistent kernel is available (tests)

    @staticmethod
    def forward(ctx, X, H0, wz, wr, wh, bz, br, bh, plan, K, wimage):
        out, stash = ops.dcrnn_seq_fwd(plan, X, wz, wr, wh, bz, br, bh, K, h0=H0, stash=True, wimage=wimage)
        ctx.plan, ctx.K, ctx.has_bias, ctx.has_h0 = plan, K, bz is not None, H0 is not None
        # the backward kernels address X / dX as dense (B,T,N,Cin): keep the contiguous copy the forward kernel read
        ctx.save_for_backward(X.contiguous(), H0, wz, wr, wh, out, stash)
        return out

    @staticmethod
    def backward(ctx, gout):
        """Reverse-time loop with 8 launches per step: [carry] -> GEMM -> 2 transposed SpMMs (in-place adjoint) -> [zr] ->
        GEMM -> 2 transposed SpMMs.  Everything that does not depend on the dH recurrence is hoisted out: both bases of
        every step are built with 4 batched SpMMs straight into their column blocks, and the weight gradients are two
        large GEMMs over all (t, b, n) rows after the loop.  Two persistent kernels replace the loop where they apply: hidden 32 / K = 2
        (`dcrnn_bwd_seq`, with its own bases and weight-gradient kernels) and narrow states, cout <= 4 (`dcrnn_narrow_bwd_seq`, after the
        same hoisted bases and before the same `_weight_grads`)."""
        X, H0, wz, wr, wh, out, stash = ctx.saved_tensors
        plan, K = ctx.plan, ctx.K
        B, T, N, Ci = X.shape
        Co = wz.size(-1)
        C = Ci + Co
        nb = 2 * K - 1
        f32 = dict(device=X.device, dtype=torch.float32)
        WhsT, WzrT = ops.dcrnn_pack_bwd_weights(wz, wr, wh, Ci, K)        # transposed stacked weights, one launch
        gout = gout.contiguous()
        if _DcrnnSeqFn.fused_backward and ops.dcrnn_bwd_supported(plan, Ci, Co, K):
            # small graph: the whole reverse recurrence is ONE persistent launch (dL/dH stays in shared memory), the bases
            # of all steps are one more, and the weight gradients are one contraction over all (t, b, n) rows
            ld = ops.dcrnn_bwd_basis_ld(Ci, Co, K)                                   # pad columns are never written nor used
            S1 = torch.empty(T * B, N, ld, **f32)
            S2 = torch.empty(T * B, N, ld, **f32)
            dph_all = torch.empty(T, B, N, Co, **f32)
            dpzr_all = torch.empty(T, B, N, 2 * Co, **f32)
            dX = torch.empty(X.shape, **f32) if ctx.needs_input_grad[0] else None   # dense: the kernels write (B,T,N,Cin) row-major
            dH0 = torch.empty(B, N, Co, **f32)
            # the bases depend only on forward results, the recurrence only on gout: run them side by side -- the
            # recurrence occupies one SM per window (64 of 132 at the reference's batch size), the basis kernel fills the
            # rest.  Fork/join with events, so a CUDA-graph capture records two parallel branches.
            main = torch.cuda.current_stream(X.device)
            side = _side_stream(X.device)
            side.wait_stream(main)
            with torch.cuda.stream(side):
                ops.dcrnn_bwd_basis(plan, X, out, H0, stash, S1, S2)
            ops.dcrnn_bwd_seq(plan, Ci, gout, out, H0, stash, WhsT, WzrT, dph_all, dpzr_all, dX, dH0)
            main.wait_stream(side)
            # weight / bias gradients over all (t, b, n) rows: per-CTA partial products + one fixed-order reduction (2 launches)
            gz, gr, gh, gbz, gbr, gbh = ops.dcrnn_bwd_wgrad(Ci, K, S1, S2, dpzr_all, dph_all, ctx.has_bias)
            gH0 = dH0 if (ctx.has_h0 and ctx.needs_input_grad[1]) else None
            return dX, gH0, gz, gr, gh, gbz, gbr, gbh, None, None, None
        Z, R, Ht = stash[:, :, 0], stash[:, :, 1], stash[:, :, 2]                          # (B,T,N,Co) strided views
        # ---- hoisted: H_{t-1} for every t (time-major so that [t] is a dense (B,N,Co) block) and both bases ------------
        Hp = torch.empty(T, B, N, Co, **f32)
        if H0 is not None:
            Hp[0] = H0
        else:
            Hp[0].zero_()
        if T > 1:
            Hp[1:] = out[:, :-1].transpose(0, 1)
        S1 = torch.empty(T * B, N, nb * C, **f32)                                          # basis of [X | H_{t-1}]
        S2 = torch.empty(T * B, N, nb * C, **f32)                                          # basis of [X | H_{t-1} * R]
        Xt = X.transpose(0, 1).reshape(T * B, N, Ci)
        S1[..., :Ci] = Xt
        S2[..., :Ci] = Xt
        S1[..., Ci:C] = Hp.view(T * B, N, Co)
        torch.mul(Hp, R.transpose(0, 1), out=S2.view(T, B, N, nb * C)[..., Ci:C])
        for S in (S1, S2):
            _x_blocks(plan, S, C, C, K, ops.spmm_cols)
        dph_all = torch.empty(T, B, N, Co, **f32)
        dpzr_all = torch.empty(T, B, N, 2 * Co, **f32)
        if _DcrnnSeqFn.fused_backward and Co <= 4 and ops.dcrnn_narrow_bwd_supported(plan, Ci, Co, K):
            # narrow states (cout <= 4): the whole reverse recurrence is ONE persistent launch, dL/dH stays on chip
            dX = torch.empty(X.shape, **f32) if ctx.needs_input_grad[0] else None
            dH0 = torch.empty(B, N, Co, **f32)
            ops.dcrnn_narrow_bwd_seq(plan, Ci, K, gout, out, H0, stash, WhsT, WzrT, dph_all, dpzr_all, dX, dH0)
            gH0 = dH0 if (ctx.has_h0 and ctx.needs_input_grad[1]) else None
            return (dX, gH0, *_weight_grads(S1, S2, dph_all, dpzr_all, K, C, Co, ctx.has_bias), None, None, None)
        # ---- the recurrence ---------------------------------------------------------------------------------------------
        buf2 = torch.empty(B, N, nb * C, **f32)                                            # dL/dS2 -> (in place) dL/d[X | H*R]
        buf1 = torch.empty(B, N, nb * C, **f32)                                            # dL/dS1 -> (in place) dL/d[X | H_{t-1}]
        g = torch.empty(B, N, Co, **f32)
        dX = torch.empty(X.shape, **f32) if ctx.needs_input_grad[0] else None   # dense: the kernels write (B,T,N,Cin) row-major
        for t in range(T - 1, -1, -1):
            if t == T - 1:
                ops.gru_bwd_carry(Ci, Co, buf2, buf1, gout=gout[:, t], z=Z[:, t], ht=Ht[:, t], g=g, dph=dph_all[t])
            else:
                ops.gru_bwd_carry(Ci, Co, buf2, buf1, g_prev=g, z_prev=Z[:, t + 1], r_prev=R[:, t + 1],
                                  dx=None if dX is None else dX[:, t + 1], gout=gout[:, t], z=Z[:, t], ht=Ht[:, t], g=g, dph=dph_all[t])
            torch.matmul(dph_all[t].view(B * N, Co), WhsT, out=buf2.view(B * N, nb * C))
            _x_blocks_adjoint(plan, buf2, C, C, K, ops.spmm_cols)
            ops.gru_bwd_zr(Ci, Co, g, Hp[t], Z[:, t], R[:, t], Ht[:, t], buf2, dpzr_all[t])
            torch.matmul(dpzr_all[t].view(B * N, 2 * Co), WzrT, out=buf1.view(B * N, nb * C))
            _x_blocks_adjoint(plan, buf1, C, C, K, ops.spmm_cols)
        dH0 = torch.empty(B, N, Co, **f32)
        ops.gru_bwd_carry(Ci, Co, buf2, buf1, g_prev=g, z_prev=Z[:, 0], r_prev=R[:, 0], dx=None if dX is None else dX[:, 0], dh_out=dH0)
        gH0 = dH0 if (ctx.has_h0 and ctx.needs_input_grad[1]) else None
        return (dX, gH0, *_weight_grads(S1, S2, dph_all, dpzr_all, K, C, Co, ctx.has_bias), None, None, None)


class _DcrnnRowsFn(torch.autograd.Function):
    """Training form of the row-split BatchedDCRNN recurrence at 32 hidden channels (H_0 = 0): forward = `stmp_dcrnn_rows_fwd` with the
    stash and the weight-gradient bases (the inference launches, so the output is bit-identical to the `no_grad` one); backward =
    `stmp_dcrnn_rows_bwd` + `stmp_dcrnn_bwd_wgrad`: dX (when X requires grad) and the gradients of the three gates' (2, 2, C, 32) weights
    and biases.  `packed` = (whsT, wzrT) of dcrnn_pack_bwd_weights for the current weights."""

    @staticmethod
    def forward(ctx, X, wz, wr, wh, bz, br, bh, plan, packed):
        whsT, wzrT = packed
        out, stash, S1, S2 = ops.dcrnn_rows_fwd(plan, X.detach(), wzrT, whsT, bz, br, bh, train=True)
        ctx.plan, ctx.K, ctx.cin, ctx.has_bias = plan, 2, X.size(-1), bz is not None
        ctx.save_for_backward(out, stash, S1, S2, whsT, wzrT)
        return out

    @staticmethod
    def backward(ctx, gout):
        out, stash, S1, S2, whsT, wzrT = ctx.saved_tensors
        dph, dpzr, dX = ops.dcrnn_rows_bwd(ctx.plan, ctx.cin, gout, out, stash, wzrT, whsT, ctx.needs_input_grad[0])
        g = _rows_param_grads(ctx, S1, 32, lambda: ops.dcrnn_bwd_wgrad(ctx.cin, 2, S1, S2, dpzr, dph, ctx.has_bias))
        return (dX, *g, None, None)


class _DcrnnHoistedRowsFn(torch.autograd.Function):
    """Training form of the narrow and 64-wide row-split BatchedDCRNN recurrences (H_0 = 0): forward = `ops.dcrnn_hoisted_rows_fwd` with
    the stash and the weight-gradient bases (the inference launches, so the output is bit-identical to the `no_grad` one); backward =
    `ops.dcrnn_hoisted_rows_bwd` (with the hoisted dX adjoint when X requires grad) and the weight / bias gradients of `_weight_grads`.
    `packed` = (whsT, wzrT) of dcrnn_pack_bwd_weights for the current weights."""

    @staticmethod
    def forward(ctx, X, wz, wr, wh, bz, br, bh, plan, K, packed):
        whsT, wzrT = packed
        out, stash, S1, S2 = ops.dcrnn_hoisted_rows_fwd(plan, X.detach(), wzrT, whsT, bz, br, bh, K, train=True)
        ctx.plan, ctx.K, ctx.cin, ctx.has_bias = plan, K, X.size(-1), bz is not None
        ctx.save_for_backward(out, stash, S1, S2, whsT, wzrT)
        return out

    @staticmethod
    def backward(ctx, gout):
        out, stash, S1, S2, whsT, wzrT = ctx.saved_tensors
        K, cin, cout = ctx.K, ctx.cin, out.size(-1)
        dph, dpzr, dX = ops.dcrnn_hoisted_rows_bwd(ctx.plan, cin, K, gout, out, stash, wzrT, whsT, ctx.needs_input_grad[0])
        g = _rows_param_grads(ctx, S1, cout, lambda: _weight_grads(S1, S2, dph, dpzr, K, cin + cout, cout, ctx.has_bias))
        return (dX, *g, None, None, None)


class DConv(torch.nn.Module):
    r"""Diffusion convolution (reference: dcrnn.py:7-111).  Messages use only the degree norms, never
    edge_weight (:39-40); norm_in is indexed by `row` and paired positionally with the re-sorted
    reverse edge list (:74-77) -- reproduced inside the plan (csrc/plan.cu)."""

    _batched_semantics = False

    def __init__(self, in_channels, out_channels, K, bias=True):
        super().__init__()
        assert K > 0
        self.in_channels = in_channels
        self.out_channels = out_channels
        self.weight = torch.nn.Parameter(torch.empty(2, K, in_channels, out_channels))
        if bias:
            self.bias = torch.nn.Parameter(torch.empty(out_channels))
        else:
            self.register_parameter("bias", None)
        self._plans = PlanCache()
        self._reset_parameters()

    def _reset_parameters(self):
        torch.nn.init.xavier_uniform_(self.weight)
        if self.bias is not None:
            torch.nn.init.zeros_(self.bias)

    def _plan(self, edge_index, edge_weight, num_nodes):
        flags = _lib.DCONV_ALLOW_DUPLICATES if self._batched_semantics else 0
        return self._plans.get(_lib.FLAVOR_DCONV, edge_index, edge_weight, num_nodes, flags=flags)

    def forward(self, X: torch.FloatTensor, edge_index: torch.LongTensor, edge_weight: torch.FloatTensor = None,
                cached_idx: bool = False) -> torch.FloatTensor:
        _require_cuda(X, "X")
        plan = self._plan(edge_index, edge_weight, X.size(-2))
        S = torch.cat(_basis(plan, X, self.weight.size(1)), dim=-1)
        H = torch.matmul(S, _stack_weight(self.weight))
        if self.bias is not None:
            H = H + self.bias
        return H


class BatchedDConv(DConv):
    """Reference: dcrnn.py:222-325 (degrees by scatter_add, duplicates legal).  `forward(X, edge_index,
    edge_weight, cached_idx)`: the plan cache subsumes `cached_idx`."""
    _batched_semantics = True


class DCRNN(torch.nn.Module):
    r"""Diffusion Convolutional GRU cell (reference: dcrnn.py:114-219).

    Args: in_channels, out_channels, K, bias -- as the reference (:128)."""

    _conv_cls = DConv
    _batched_semantics = False
    _fused_training = True   # training forward = fused kernel + stash, backward = hand-written reverse-time loop

    def __init__(self, in_channels: int, out_channels: int, K: int, bias: bool = True):
        super().__init__()
        self.in_channels = in_channels
        self.out_channels = out_channels
        self.K = K
        self.bias = bias
        C = in_channels + out_channels
        self.conv_x_z = self._conv_cls(C, out_channels, K, bias)
        self.conv_x_r = self._conv_cls(C, out_channels, K, bias)
        self.conv_x_h = self._conv_cls(C, out_channels, K, bias)
        self._plans = PlanCache()
        self._wimg = ops.PackCache()

    # ---- helpers -----------------------------------------------------------------------------------
    def _plan(self, edge_index, edge_weight, num_nodes):
        flags = _lib.DCONV_ALLOW_DUPLICATES if self._batched_semantics else 0
        return self._plans.get(_lib.FLAVOR_DCONV, edge_index, edge_weight, num_nodes, flags=flags)

    def _needs_grad(self, *tensors):
        if not torch.is_grad_enabled():
            return False
        return any(p.requires_grad for p in self.parameters()) or any(t is not None and t.requires_grad for t in tensors)

    def _params(self):
        return (self.conv_x_z.weight, self.conv_x_r.weight, self.conv_x_h.weight,
                self.conv_x_z.bias, self.conv_x_r.bias, self.conv_x_h.bias)

    def _weight_image(self):
        """B-operand image for the wgmma kernel, rebuilt only when a parameter changes."""
        return self._wimg.get(list(self.parameters()),
                              lambda: ops.dcrnn_weight_image(*self._params(), self.in_channels, self.K))

    def _tiled_step(self, plan, X, H):
        """One GRU step on (N,*) or (B,N,*) tensors; z and r share the diffusion of [X|H]."""
        wz, wr, wh, bz, br, bh = self._params()
        O = self.out_channels
        S = torch.cat(_basis(plan, torch.cat([X, H], dim=-1), self.K), dim=-1)
        pre = torch.matmul(S, torch.cat([_stack_weight(wz), _stack_weight(wr)], dim=1))
        if bz is not None:
            pre = pre + torch.cat([bz, br])
        Z, R = torch.sigmoid(pre[..., :O]), torch.sigmoid(pre[..., O:])
        S2 = torch.cat(_basis(plan, torch.cat([X, H * R], dim=-1), self.K), dim=-1)
        ph = torch.matmul(S2, _stack_weight(wh))
        if bh is not None:
            ph = ph + bh
        Ht = torch.tanh(ph)
        return Z * H + (1 - Z) * Ht

    # ---- reference surface -------------------------------------------------------------------------
    def forward(self, X: torch.FloatTensor, edge_index: torch.LongTensor, edge_weight: torch.FloatTensor = None,
                H: torch.FloatTensor = None) -> torch.FloatTensor:
        """X (N,Cin), H (N,Cout) or None -> H' (N,Cout)   (dcrnn.py:194-219)."""
        _require_cuda(X, "X")
        N = X.shape[0]
        plan = self._plan(edge_index, edge_weight, N)
        if not self._needs_grad(X, H) and ops.dcrnn_seq_supported(plan, self.in_channels, self.out_channels, self.K):
            h0 = None if H is None else H.reshape(1, N, self.out_channels)
            out = ops.dcrnn_seq_fwd(plan, X.reshape(1, 1, N, self.in_channels), *self._params(), self.K, h0=h0,
                                    wimage=self._weight_image())
            return out[0, 0]
        if self._fused_training and ops.dcrnn_seq_supported(plan, self.in_channels, self.out_channels, self.K):
            h0 = None if H is None else H.reshape(1, N, self.out_channels)
            return _DcrnnSeqFn.apply(X.reshape(1, 1, N, self.in_channels), h0, *self._params(), plan, self.K, self._weight_image())[0, 0]
        if H is None:
            H = torch.zeros(N, self.out_channels, device=X.device, dtype=X.dtype)
        return self._tiled_step(plan, X, H)


class BatchedDCRNN(DCRNN):
    """Batched seq-to-seq DCRNN (reference: dcrnn.py:328-475).  X (B,T,N,Cin) -> (B,T,N,Cout), H_0 = 0.
    The reference replicates the graph B times block-diagonally (:363-369); the block-diagonal operator
    equals the single-graph operator applied per window, so nothing is replicated here."""

    _conv_cls = BatchedDConv
    _batched_semantics = True

    def __init__(self, in_channels: int, out_channels: int, K: int, bias: bool = True):
        super().__init__(in_channels, out_channels, K, bias)
        self._rows_pack = ops.PackCache()

    def _rows_ok(self, plan, X, training):
        """The row-split routes (`ops.dcrnn_rows_supported`: in_channels 1..4 and out_channels = 32 at K = 2, out_channels and K in 1..4, or
        out_channels = 64 at K = 2 or 3): float32 X, `_fused_training` for training calls and a graph the one-SM kernels cannot hold.  The
        envelope is checked on the module's attributes before the library is consulted, so other shapes never consult it."""
        if X.dtype != torch.float32 or (training and not self._fused_training):
            return False
        cin, cout, K = self.in_channels, self.out_channels, self.K
        return ops.dcrnn_rows_supported(plan, cin, cout, K) and not ops.dcrnn_seq_supported(plan, cin, cout, K)

    def _rows_packed(self):
        """(whsT, wzrT) of dcrnn_pack_bwd_weights for the row-split kernels, rebuilt only when a parameter changes."""
        return self._rows_pack.get(list(self.parameters()),
                                   lambda: ops.dcrnn_pack_bwd_weights(*self._params()[:3], self.in_channels, self.K))

    def _rows_infer(self, plan, x, **window):
        """A no_grad call on the row-split kernels: the 32-wide ones read the windows in place (also at `win_start`), the narrow and
        64-wide ones diffuse X once up front (`ops.dcrnn_hoisted_rows_fwd`, windows at `win_start` gathered into the hoisted X blocks)."""
        whsT, wzrT = self._rows_packed()
        if self.out_channels == 32:
            return ops.dcrnn_rows_fwd(plan, x, wzrT, whsT, *self._params()[3:], **window)
        return ops.dcrnn_hoisted_rows_fwd(plan, x, wzrT, whsT, *self._params()[3:], self.K, **window)

    def forward(self, X, edge_index, edge_weight):
        _require_cuda(X, "X")
        B, T, N, F = X.size()
        plan = self._plan(edge_index, edge_weight, N)
        if not self._needs_grad(X) and ops.dcrnn_seq_supported(plan, self.in_channels, self.out_channels, self.K):
            try:
                return ops.dcrnn_seq_fwd(plan, X, *self._params(), self.K, wimage=self._weight_image())
            except _lib.StmpUnsupported:
                pass
        if self._fused_training and ops.dcrnn_seq_supported(plan, self.in_channels, self.out_channels, self.K):
            try:
                return _DcrnnSeqFn.apply(X, None, *self._params(), plan, self.K, self._weight_image())
            except _lib.StmpUnsupported:
                pass
        training = self._needs_grad(X)
        if self._rows_ok(plan, X, training):    # graphs larger than one SM, or 64 hidden channels: all windows of a step per launch
            if not training:
                return self._rows_infer(plan, X)
            if self.out_channels == 32:
                return _DcrnnRowsFn.apply(X, *self._params(), plan, self._rows_packed())
            return _DcrnnHoistedRowsFn.apply(X, *self._params(), plan, self.K, self._rows_packed())
        H = torch.zeros(B, N, self.out_channels, device=X.device, dtype=X.dtype)
        outs = []
        for t in range(T):
            H = self._tiled_step(plan, X[:, t], H)
            outs.append(H)
        return torch.stack(outs, dim=1)

    def forward_indexed(self, series, win_start, horizon, edge_index, edge_weight):
        """Index-batching entry: windows are read in-kernel from the resident series (T_total,N,Cin)
        at `win_start` (int64 [B]) -- the fused form of IndexDataset + DataLoader collate + forward."""
        _require_cuda(series, "series")
        plan = self._plan(edge_index, edge_weight, series.size(1))
        if not self._needs_grad(series) and ops.dcrnn_seq_supported(plan, self.in_channels, self.out_channels, self.K):
            try:
                return ops.dcrnn_seq_fwd(plan, series, *self._params(), self.K, win_start=win_start, horizon=horizon,
                                         wimage=self._weight_image())
            except _lib.StmpUnsupported:      # e.g. a horizon whose shared-memory layout the FFMA kernel cannot hold
                pass
        if not self._needs_grad(series) and self._rows_ok(plan, series, False):
            return self._rows_infer(plan, series, win_start=win_start, horizon=horizon)
        X = ops.window_gather(series, win_start, horizon, with_target=False)
        return self.forward(X, edge_index, edge_weight)
