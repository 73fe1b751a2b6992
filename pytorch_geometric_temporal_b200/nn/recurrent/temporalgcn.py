"""TGCN / TGCN2 -- drop-in for torch_geometric_temporal/nn/recurrent/temporalgcn.py (:5-130, :133-233).
state_dict keys `conv_{z,r,h}.lin.weight (out,in)`, `conv_{z,r,h}.bias`, `linear_{z,r,h}.{weight,bias}`.
The reference runs three GCNConvs (each: gcn_norm + lin + propagate of `out` channels); since
A^(X W) = (A^ X) W, one SpMM on the `in` channels feeds all three gates."""
import math

import torch

from ... import _lib, ops
from ...plan import PlanCache, _require_cuda
from ._cheb import _Lin


class GCNParams(torch.nn.Module):
    """Holder with GCNConv's keys: `lin.weight (out,in)` glorot, `bias (out)` zeros."""

    def __init__(self, in_channels, out_channels):
        super().__init__()
        self.lin = _Lin(in_channels, out_channels)
        self.bias = torch.nn.Parameter(torch.zeros(out_channels))


class TGCN(torch.nn.Module):
    def __init__(self, in_channels: int, out_channels: int, improved: bool = False, cached: bool = False,
                 add_self_loops: bool = True):
        super().__init__()
        self.in_channels, self.out_channels = in_channels, out_channels
        self.improved, self.cached, self.add_self_loops = improved, cached, add_self_loops
        for g in "zrh":  # creation order as the reference: conv then linear, per gate (:36-76)
            setattr(self, f"conv_{g}", GCNParams(in_channels, out_channels))
            setattr(self, f"linear_{g}", torch.nn.Linear(2 * out_channels, out_channels))
        self._plans = PlanCache()
        self._pack = ops.PackCache()

    def _plan(self, edge_index, edge_weight, num_nodes):
        flags = (_lib.GCN_IMPROVED if self.improved else 0) | (0 if self.add_self_loops else _lib.GCN_NO_SELF_LOOPS)
        return self._plans.get(_lib.FLAVOR_GCN, edge_index, edge_weight, num_nodes, flags=flags)

    def _gcn_all(self, plan, X):
        """[GCN_z(X) | GCN_r(X) | GCN_h(X)] = (A^ X) [Wz|Wr|Wh]^T + [bz|br|bh]."""
        AX = ops.spmm(plan, 0, X)
        W = torch.cat([self.conv_z.lin.weight, self.conv_r.lin.weight, self.conv_h.lin.weight], dim=0)
        b = torch.cat([self.conv_z.bias, self.conv_r.bias, self.conv_h.bias])
        return torch.nn.functional.linear(AX, W, b)

    def _cell(self, G, H):
        Co = self.out_channels
        Gz, Gr, Gh = G[..., :Co], G[..., Co:2 * Co], G[..., 2 * Co:]
        lin = lambda l, a, b: torch.matmul(a, l.weight[:, :Co].t()) + torch.matmul(b, l.weight[:, Co:].t()) + l.bias
        Z = torch.sigmoid(lin(self.linear_z, Gz, H))
        R = torch.sigmoid(lin(self.linear_r, Gr, H))
        Ht = torch.tanh(lin(self.linear_h, Gh, H * R))
        return Z * H + (1 - Z) * Ht

    def _packed(self):
        """Fold GCNConv (lin, bias) and the gate Linear into the fused kernel's layout:
        pre_g = H' @ L2^T + (A^X) @ (L1 W)^T + (L1 b + l),  L = linear_g.weight = [L1 | L2]."""
        def build():
            Ci, Co, dev = self.in_channels, self.out_channels, self.conv_z.lin.weight.device
            W = torch.zeros(96, 112, device=dev)
            b = torch.zeros(96, device=dev)
            for gi, g in enumerate("zrh"):
                conv, lin = getattr(self, f"conv_{g}"), getattr(self, f"linear_{g}")
                L1, L2 = lin.weight[:, :Co], lin.weight[:, Co:]
                r = slice(32 * gi, 32 * gi + 32)
                W[r, 0:32] = L2
                W[r, 100:100 + Ci] = L1 @ conv.lin.weight
                b[r] = L1 @ conv.bias + lin.bias
            return W, b, ops.gru_weight_image(W, b)
        return self._pack.get(list(self.parameters()), build)

    def _packed3(self):
        """The same folding for `stmp_tgcn_attn_fwd` (any graph size):  pre_g = (A^X) A[:, g] + H' Bm[:, g] + c[g]
        with A = (L1 W)^T (in x out), Bm = L2^T (out x out), c = L1 b + l;  columns z | r | h, each a block of the kernel's width:
        64 columns at out_channels = 64 (the *_wide_* entries), 32 otherwise."""
        def build():
            Ci, Co, dev = self.in_channels, self.out_channels, self.conv_z.lin.weight.device
            w = 64 if Co == 64 else 32
            A = torch.zeros(Ci, 3 * w, device=dev)
            Bm = torch.zeros(w, 3 * w, device=dev)
            c = torch.zeros(3 * w, device=dev)
            for gi, g in enumerate("zrh"):
                conv, lin = getattr(self, f"conv_{g}"), getattr(self, f"linear_{g}")
                L1, L2 = lin.weight[:, :Co], lin.weight[:, Co:]
                r = slice(w * gi, w * gi + Co)
                A[:, r] = (L1 @ conv.lin.weight).t()
                Bm[:Co, r] = L2.t()
                c[r] = L1 @ conv.bias + lin.bias
            return A, Bm, c
        if not hasattr(self, "_pack3"):
            self._pack3 = ops.PackCache()
        return self._pack3.get(list(self.parameters()), build)

    def _fold3(self):
        """`_packed3` without the cache, as differentiable torch ops (the training path: the gradients of the folded weights flow back to
        conv_g.lin.weight, conv_g.bias and linear_g through autograd on these few small matrices)."""
        Ci, Co = self.in_channels, self.out_channels
        As, Bs, cs = [], [], []
        for g in "zrh":
            conv, lin = getattr(self, f"conv_{g}"), getattr(self, f"linear_{g}")
            L1, L2 = lin.weight[:, :Co], lin.weight[:, Co:]
            As.append((L1 @ conv.lin.weight).t())
            Bs.append(L2.t())
            cs.append(L1 @ conv.bias + lin.bias)
        return torch.cat(As, dim=1), torch.cat(Bs, dim=1), torch.cat(cs)

    # The fused kernels take the batch rows as the grid's y dimension, so at most 65 535 of them; a larger batch takes the op-for-op path.
    _FUSED_MAX_ROWS = 65535
    # hidden widths the fused temporal-attention kernels and their backwards serve
    _ATTN_WIDTHS = (32, 64)

    def _attn_train_ok(self, X, H, periods, rows):
        """The fused kernel pair (forward + hand-written backward) trains the configuration of the reference's examples: no incoming state,
        no gradient w.r.t. X, out_channels 32 or 64, in_channels <= 4, in_channels * periods <= 128, `rows` <= 65 535 batch rows."""
        return (H is None and torch.is_grad_enabled() and not X.requires_grad and self.out_channels in self._ATTN_WIDTHS
                and self.in_channels <= 4 and self.in_channels * periods <= 128 and rows <= self._FUSED_MAX_ROWS and self.fused_training)

    def _cell_train_ok(self, X, H):
        """The steps after the first of a training loop that carries the state (the reference's BatchedTGCN, tgcn_example.py): the
        same forward launch with H + the hand-written cell backward (dH and the folded-weight gradients).  No gradient w.r.t. X,
        out_channels 32 or 64, in_channels <= 4, H of shape X.shape[:-1] + (out_channels,), at most 65 535 batch rows."""
        return (H is not None and torch.is_grad_enabled() and not X.requires_grad and self.out_channels in self._ATTN_WIDTHS
                and self.in_channels <= 4 and tuple(H.shape) == tuple(X.shape[:-1]) + (self.out_channels,)
                and math.prod(X.shape[:-2]) <= self._FUSED_MAX_ROWS and self.fused_training)

    fused_training = True     # False: train through autograd over SpMM + cuBLAS (tests compare the two)

    def _no_grad_needed(self, X, H, *extra):
        if not torch.is_grad_enabled():
            return True
        ts = list(self.parameters()) + [X] + ([] if H is None else [H]) + list(extra)
        return not any(t.requires_grad for t in ts)

    def _attn_ok(self, X, H, periods, rows, *extra):
        """The fused temporal-attention + GCN kernel serves inference for out_channels 32 or 64, in_channels <= 4,
        in_channels * periods <= 128 and `rows` <= 65 535 batch rows on graphs of any size."""
        return (self.out_channels in self._ATTN_WIDTHS and self.in_channels <= 4 and self.in_channels * periods <= 128
                and rows <= self._FUSED_MAX_ROWS and self._no_grad_needed(X, H, *extra))

    def _fused_ok(self, plan, X, H):
        if self.out_channels != 32:
            return False
        if torch.is_grad_enabled() and (any(p.requires_grad for p in self.parameters()) or X.requires_grad
                                        or (H is not None and H.requires_grad)):
            return False
        return ops.gru_seq_supported(plan, 1, self.in_channels, self.out_channels)

    def forward(self, X: torch.FloatTensor, edge_index: torch.LongTensor, edge_weight: torch.FloatTensor = None,
                H: torch.FloatTensor = None) -> torch.FloatTensor:
        _require_cuda(X, "X")
        plan = self._plan(edge_index, edge_weight, X.size(-2))
        rows = math.prod(X.shape[:-2])
        if self._attn_ok(X, H, 1, rows):       # one period, weight 1: the cell itself
            A, Bm, c = self._packed3()
            N, Ci = X.shape[-2], X.shape[-1]
            h = None if H is None else H.reshape(-1, N, self.out_channels)
            out = ops.tgcn_attn_fwd(plan, X.reshape(-1, N, Ci, 1), A, Bm, c, None, h)
            return out.reshape(*X.shape[:-1], self.out_channels)
        if self._attn_train_ok(X, H, 1, rows):
            A, Bm, c = self._fold3()
            N, Ci = X.shape[-2], X.shape[-1]
            out = ops.tgcn_attn_train(plan, X.reshape(-1, N, Ci, 1), A, Bm, c, None)
            return out.reshape(*X.shape[:-1], self.out_channels)
        if self._cell_train_ok(X, H):
            A, Bm, c = self._fold3()
            N, Ci = X.shape[-2], X.shape[-1]
            out = ops.tgcn_cell_train(plan, X.reshape(-1, N, Ci, 1), H.reshape(-1, N, self.out_channels), A, Bm, c)
            return out.reshape(*X.shape[:-1], self.out_channels)
        if H is None:
            H = torch.zeros(*X.shape[:-1], self.out_channels, device=X.device, dtype=X.dtype)
        if self._fused_ok(plan, X, H):   # every (batch) row is an independent 1-step window of the fused kernel
            W, b, img = self._packed()
            N, Ci = X.shape[-2], X.shape[-1]
            out = ops.gru_seq_fwd(plan, 1, X.reshape(-1, 1, N, Ci), W, b, h0=H.reshape(-1, N, self.out_channels), wimage=img)
            return out.reshape(*X.shape[:-1], self.out_channels)
        return self._cell(self._gcn_all(plan, X), H)


class TGCN2(TGCN):
    """Batched variant (temporalgcn.py:133-233): X (B,N,F), H (B,N,out); `batch_size` kept for signature
    compatibility only (as in the reference, :147-148)."""

    def __init__(self, in_channels: int, out_channels: int, batch_size: int, improved: bool = False, cached: bool = False,
                 add_self_loops: bool = True):
        super().__init__(in_channels, out_channels, improved, cached, add_self_loops)
        self.batch_size = batch_size
