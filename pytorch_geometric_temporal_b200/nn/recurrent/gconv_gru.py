"""GConvGRU -- drop-in for torch_geometric_temporal/nn/recurrent/gconv_gru.py (:5-170): same
constructor `(in_channels, out_channels, K, normalization="sym", bias=True)`, `forward(X, edge_index,
edge_weight=None, H=None, lambda_max=None)`, state_dict keys `conv_{x,h}_{z,r,h}.lins.{k}.weight`,
`.bias`.  The six ChebConvs of the reference renormalise the graph and re-propagate per gate; here the
scaled Laplacian is a cached plan and T_k([X|H]) is computed once and shared by all gates.

Inside the fused envelope (K <= 2, out_channels = 32, in_channels <= 4, a graph that fits one SM) inference is one launch of the
generic graph-GRU kernel, and training is that same launch plus a hand-written backward (ops.gru_seq_train): the gradients of the
prepacked weights are handed to the parameters as blocks, so the cached fold needs no autograd graph.  Graphs too large for one SM
(K <= 2, out_channels = 32, in_channels <= 16, 2-D X) run the row-split cell kernels instead (ops.gru_rows_fwd / gru_rows_train):
one launch with H = None, two with H given, and a hand-written backward of the same kind.  At out_channels = 64 (K <= 2, in_channels <=
16, 2-D X) every graph, small or large, runs the 64-wide instance of those kernels (stmp_gru_wide_rows_*): no one-SM kernel holds that
width."""
import torch

from ... import ops
from ...plan import _require_cuda
from ._cheb import ChebParams, ChebPlanMixin, broadcast_states, cheb_basis


class GConvGRU(torch.nn.Module, ChebPlanMixin):
    def __init__(self, in_channels: int, out_channels: int, K: int, normalization: str = "sym", bias: bool = True):
        super().__init__()
        self.in_channels, self.out_channels, self.K = in_channels, out_channels, K
        self.normalization, self.bias = normalization, bias
        for g in "zrh":
            setattr(self, f"conv_x_{g}", ChebParams(in_channels, out_channels, K, bias))
            setattr(self, f"conv_h_{g}", ChebParams(out_channels, out_channels, K, bias))
        self._init_plans()
        self._pack = ops.PackCache()
        self._rows_pack = ops.PackCache()
        self.fused_training = True      # False: op-for-op autograd path (tests compare the two)

    def _gate_weight(self, g, x_only=False, h_only=False):
        """Rows follow the basis [T_0 | T_1 | ...] of U=[X|H]: block k = [Wx_k^T ; Wh_k^T]."""
        cx, ch = getattr(self, f"conv_x_{g}"), getattr(self, f"conv_h_{g}")
        rows = []
        for k in range(self.K):
            if not h_only:
                rows.append(cx.lins[k].weight.t())
            if not x_only:
                rows.append(ch.lins[k].weight.t())
        return torch.cat(rows, dim=0)

    def _gate_bias(self, g):
        cx, ch = getattr(self, f"conv_x_{g}"), getattr(self, f"conv_h_{g}")
        return None if cx.bias is None else cx.bias + ch.bias

    def _packed(self):
        """(wcat [96,112], bcat [96]) for stmp_gru_seq_fwd: columns H | L^H | - | X | L^X | - (one operator)."""
        def build():
            Ci, dev = self.in_channels, self.conv_x_z.lins[0].weight.device
            W = torch.zeros(96, 112, device=dev)
            b = torch.zeros(96, device=dev)
            for gi, g in enumerate("zrh"):
                cx, ch = getattr(self, f"conv_x_{g}"), getattr(self, f"conv_h_{g}")
                r = slice(32 * gi, 32 * gi + 32)
                W[r, 0:32] = ch.lins[0].weight
                W[r, 96:96 + Ci] = cx.lins[0].weight
                if self.K > 1:
                    W[r, 32:64] = ch.lins[1].weight
                    W[r, 100:100 + Ci] = cx.lins[1].weight
                if cx.bias is not None:
                    b[r] = cx.bias + ch.bias
            return W, b, ops.gru_weight_image(W, b)
        return self._pack.get(list(self.parameters()), build)

    def _rows_packed(self):
        """(w [3 Co, K(Ci+Co)], b [3 Co]) for stmp_gru_rows_fwd / stmp_gru_wide_rows_fwd: columns [X | H] per Chebyshev order (one launch per
        weight update)."""
        def build():
            gates = [(getattr(self, f"conv_x_{g}"), getattr(self, f"conv_h_{g}")) for g in "zrh"]
            wx = torch.stack([torch.stack([cx.lins[k].weight for k in range(self.K)]) for cx, _ in gates])
            wh = torch.stack([torch.stack([ch.lins[k].weight for k in range(self.K)]) for _, ch in gates])
            bx = bh = None
            if self.bias:
                bx, bh = torch.stack([cx.bias for cx, _ in gates]), torch.stack([ch.bias for _, ch in gates])
            return ops.gru_rows_pack_weights(self.K - 1, self.in_channels, wx, wh, bx, bh)
        return self._rows_pack.get(list(self.parameters()), build)

    def _param_spec(self, rows=False):
        """(spec, params) of ops.gru_seq_train (or, with `rows`, ops.gru_rows_train): where each parameter's gradient sits in the packed
        weight / bias gradients -- the inverse of `_packed` (`_rows_packed`).  Both ChebConvs of a gate add their biases, so both receive
        that gate's bias block."""
        spec, params = [], []
        Ci, Co = self.in_channels, (self.out_channels if rows else 32)
        for gi, g in enumerate("zrh"):
            cx, ch = getattr(self, f"conv_x_{g}"), getattr(self, f"conv_h_{g}")
            for k in range(self.K):
                spec.append(("w", Co * gi, Co, k * (Ci + Co) + Ci if rows else 32 * k, Co))
                params.append(ch.lins[k].weight)
                spec.append(("w", Co * gi, Co, k * (Ci + Co) if rows else 96 + 4 * k, Ci))
                params.append(cx.lins[k].weight)
            if cx.bias is not None:
                spec += [("b", Co * gi, Co), ("b", Co * gi, Co)]
                params += [cx.bias, ch.bias]
        return spec, params

    def _train_ok(self, plan, X, H):
        """The fused training route: grad enabled and something requires it, inside the envelope of both the forward and the
        backward kernels for n_ops = K - 1."""
        if not self.fused_training or self.K > 2 or self.out_channels != 32 or self.in_channels > 4 or X.dim() != 2:
            return False
        if not (torch.is_grad_enabled() and (any(p.requires_grad for p in self.parameters()) or X.requires_grad or H.requires_grad)):
            return False
        if H.shape != (X.size(0), 32) or X.dtype != torch.float32 or H.dtype != torch.float32:
            return False
        n_ops = self.K - 1
        return (ops.gru_seq_supported(plan, n_ops, self.in_channels, self.out_channels)
                and ops.gru_bwd_supported(plan, n_ops, self.in_channels, self.out_channels))

    def _fused_ok(self, plan, X, H):
        if self.K > 2 or self.out_channels != 32 or X.dim() != 2:
            return False
        if torch.is_grad_enabled() and (any(p.requires_grad for p in self.parameters()) or X.requires_grad
                                        or (H is not None and H.requires_grad)):
            return False
        return ops.gru_seq_supported(plan, 1 if self.K > 1 else 0, self.in_channels, self.out_channels)

    def _rows_ok(self, plan, X, H, training):
        """The row-split route: K <= 2, out_channels 32 or 64, in_channels <= 16, 2-D float32 X; at 32 only a graph the one-SM kernel
        cannot hold (checked first, so graphs that fit one SM never consult the row-split entry), at 64 any graph; training calls also need
        `fused_training`."""
        Co = self.out_channels
        if self.K > 2 or Co not in (32, 64) or self.in_channels > 16 or X.dim() != 2 or X.dtype != torch.float32:
            return False
        if (training and not self.fused_training) or (H is not None and (H.shape != (X.size(0), Co) or H.dtype != torch.float32)):
            return False
        n_ops = self.K - 1
        if Co == 32 and ops.gru_seq_supported(plan, n_ops, 1, 32):
            return False
        return ops.gru_rows_supported(plan, n_ops, self.in_channels, Co)

    def forward(self, X: torch.FloatTensor, edge_index: torch.LongTensor, edge_weight: torch.FloatTensor = None,
                H: torch.FloatTensor = None, lambda_max: torch.Tensor = None) -> torch.FloatTensor:
        _require_cuda(X, "X")
        N, Ci, Co, K = X.size(-2), self.in_channels, self.out_channels, self.K
        H_given = H
        if H is None:
            H = torch.zeros(*X.shape[:-1], Co, device=X.device, dtype=X.dtype)
        plan = self._cheb_plan(edge_index, edge_weight, N, self.normalization, lambda_max)
        if self._fused_ok(plan, X, H):   # one wgmma launch for the whole cell (stmp_gru_seq_fwd)
            W, b, img = self._packed()
            return ops.gru_seq_fwd(plan, 1 if K > 1 else 0, X.reshape(1, 1, N, Ci), W, b, h0=H.reshape(1, N, Co), wimage=img)[0, 0]
        if self._train_ok(plan, X, H):   # the same launch with a stash, and a hand-written backward
            W, b, img = self._packed()
            spec, params = self._param_spec()
            h0 = None if H_given is None else H_given.reshape(1, N, Co)      # None: zeros, and no dH
            return ops.gru_seq_train(plan, K - 1, X.reshape(1, 1, N, Ci), h0, W, b, img, spec, params)[0, 0]
        training = torch.is_grad_enabled() and (any(p.requires_grad for p in self.parameters()) or X.requires_grad
                                                 or (H_given is not None and H_given.requires_grad))
        if self._rows_ok(plan, X, H_given, training):   # graphs larger than one SM, or 64 channels: the row-split cell kernels
            w, b = self._rows_packed()
            if training:
                spec, params = self._param_spec(rows=True)
                return ops.gru_rows_train(plan, K - 1, X, H_given, w, b, spec, params)
            return ops.gru_rows_fwd(plan, K - 1, X, H_given, w, b)
        X, (H,) = broadcast_states(X, (H,), Co)
        TU = cheb_basis(plan, torch.cat([X, H], dim=-1), K)              # K x (N, Ci+Co)
        S = torch.cat(TU, dim=-1)
        pre = torch.matmul(S, torch.cat([self._gate_weight("z"), self._gate_weight("r")], dim=1))
        bz, br = self._gate_bias("z"), self._gate_bias("r")
        if bz is not None:
            pre = pre + torch.cat([bz, br])
        grad = torch.is_grad_enabled() and (pre.requires_grad or H.requires_grad)
        if grad:
            Z, R = torch.sigmoid(pre[..., :Co]), torch.sigmoid(pre[..., Co:])
            HR = H * R
        else:
            Z, R, HR = ops.gru_zr(pre[..., :Co].contiguous(), pre[..., Co:].contiguous(), H)
        Sx = torch.cat([t[..., :Ci] for t in TU], dim=-1)                   # T_k(X) is shared with the candidate
        Shr = torch.cat(cheb_basis(plan, HR, K), dim=-1)
        ph = torch.matmul(Sx, self._gate_weight("h", x_only=True)) + torch.matmul(Shr, self._gate_weight("h", h_only=True))
        bh = self._gate_bias("h")
        if bh is not None:
            ph = ph + bh
        if grad:
            return Z * H + (1 - Z) * torch.tanh(ph)
        return ops.gru_out(ph, Z, H)
