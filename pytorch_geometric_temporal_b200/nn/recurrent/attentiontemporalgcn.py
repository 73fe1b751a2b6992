"""A3TGCN / A3TGCN2 -- drop-in for nn/recurrent/attentiontemporalgcn.py (:7-79, :83-157).
state_dict keys `_attention (periods)`, `_base_tgcn.*`.  The reference loops over the periods in Python
(12 x 3 GCNConv chains, strided X[..., p] slices); the periods are independent (the SAME H enters each,
:155), so all of them go through ONE batched SpMM + one set of GEMMs and the softmax-weighted sum."""
import math

import torch

from ... import ops
from .temporalgcn import TGCN, TGCN2
from ...plan import _require_cuda


class _A3Base(torch.nn.Module):
    def _forward_all_periods(self, X, edge_index, edge_weight, H):
        _require_cuda(X, "X")
        base = self._base_tgcn
        P = X.shape[-1]
        rows = math.prod(X.shape[:-3])
        if base._attn_ok(X, H, P, rows, self._attention):
            # ONE launch: gather A^X for all periods per node, the GRU gates of every period and the softmax-weighted sum
            N, F = X.shape[-3], X.shape[-2]
            plan = base._plan(edge_index, edge_weight, N)
            A, Bm, c = base._packed3()
            probs = torch.nn.functional.softmax(self._attention.detach(), dim=0)
            if X.dim() == 3:                                        # A3TGCN: (N,F,P), H (N,out)
                return ops.tgcn_attn_fwd(plan, X.unsqueeze(0), A, Bm, c, probs, H, h_shared=True)[0]
            return ops.tgcn_attn_fwd(plan, X, A, Bm, c, probs, H)   # A3TGCN2: (B,N,F,P), H (B,N,out)
        if base._attn_train_ok(X, H, P, rows):
            # training without an incoming state: the same launch + a hand-written backward (gates recomputed, gradients of the folded
            # weights and of the attention probabilities reduced on the device)
            N, F = X.shape[-3], X.shape[-2]
            plan = base._plan(edge_index, edge_weight, N)
            A, Bm, c = base._fold3()
            probs = torch.nn.functional.softmax(self._attention, dim=0)
            if X.dim() == 3:
                return ops.tgcn_attn_train(plan, X.unsqueeze(0), A, Bm, c, probs)[0]
            return ops.tgcn_attn_train(plan, X, A, Bm, c, probs)
        # (..., N, F, P) -> (P, ..., N, F): periods become the leading batch axis of the SpMM
        Xp = X.movedim(-1, 0).contiguous()
        lead = Xp.shape[:-2]
        N, F = Xp.shape[-2:]
        plan = base._plan(edge_index, edge_weight, N)
        probs = torch.nn.functional.softmax(self._attention, dim=0)
        if base._fused_ok(plan, X, H) and not (torch.is_grad_enabled() and self._attention.requires_grad):
            # all periods x batch rows = independent 1-step windows of ONE fused launch; H is shared by the periods
            W, b, img = base._packed()
            Xw = Xp.reshape(-1, 1, N, F)
            if H is None:
                Hn = ops.gru_seq_fwd(plan, 1, Xw, W, b, wimage=img)
            elif X.dim() == 3:                                      # A3TGCN: a single (N,out) state for every period
                Hn = ops.gru_seq_fwd(plan, 1, Xw, W, b, h0=H, h0_shared=True, wimage=img)
            else:                                                   # A3TGCN2: (B,N,out) repeated over the periods
                Hn = ops.gru_seq_fwd(plan, 1, Xw, W, b, h0=H.unsqueeze(0).expand(P, *H.shape).reshape(-1, N, base.out_channels), wimage=img)
            Hn = Hn.reshape(*lead, N, base.out_channels)
            return torch.tensordot(probs, Hn, dims=([0], [0]))
        G = base._gcn_all(plan, Xp.reshape(-1, N, F)).reshape(*lead, N, 3 * base.out_channels)
        if H is None:
            H = torch.zeros(*X.shape[:-2], base.out_channels, device=X.device, dtype=X.dtype)
        Hn = base._cell(G, H)                                   # H broadcasts over the period axis
        return torch.tensordot(probs, Hn, dims=([0], [0]))      # sum_p probs[p] * H_p   (:153-155)


class A3TGCN(_A3Base):
    def __init__(self, in_channels: int, out_channels: int, periods: int, improved: bool = False, cached: bool = False,
                 add_self_loops: bool = True):
        super().__init__()
        self.in_channels, self.out_channels, self.periods = in_channels, out_channels, periods
        self.improved, self.cached, self.add_self_loops = improved, cached, add_self_loops
        self._base_tgcn = TGCN(in_channels, out_channels, improved, cached, add_self_loops)
        # the reference picks the device of `_attention` at construction (:48-49); a Parameter moved by
        # .to()/.cuda() with the module is equivalent and keeps state_dict compatibility
        self._attention = torch.nn.Parameter(torch.empty(periods))
        torch.nn.init.uniform_(self._attention)

    def forward(self, X, edge_index, edge_weight=None, H=None):
        return self._forward_all_periods(X, edge_index, edge_weight, H)


class A3TGCN2(_A3Base):
    def __init__(self, in_channels: int, out_channels: int, periods: int, batch_size: int, improved: bool = False,
                 cached: bool = False, add_self_loops: bool = True):
        super().__init__()
        self.in_channels, self.out_channels, self.periods, self.batch_size = in_channels, out_channels, periods, batch_size
        self.improved, self.cached, self.add_self_loops = improved, cached, add_self_loops
        self._base_tgcn = TGCN2(in_channels, out_channels, batch_size, improved, cached, add_self_loops)
        self._attention = torch.nn.Parameter(torch.empty(periods))
        torch.nn.init.uniform_(self._attention)

    def forward(self, X, edge_index, edge_weight=None, H=None):
        return self._forward_all_periods(X, edge_index, edge_weight, H)
