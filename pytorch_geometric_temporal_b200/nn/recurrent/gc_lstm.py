"""GCLSTM -- drop-in for torch_geometric_temporal/nn/recurrent/gc_lstm.py (:9-205; SURVEY 8f rank 1): constructor
`(in_channels, out_channels, K, normalization="sym", bias=True)`, `forward(X, edge_index, edge_weight, H, C,
lambda_max) -> (H, C)`, state_dict keys `conv_{i,f,c,o}.lins.{k}.weight/.bias`, `W_{i,f,c,o} (in,out)` (glorot),
`b_{i,f,c,o} (1,out)` (zeros).

The reference runs four ChebConvs on the same H (4(K-1) propagations) and four `X @ W_g` products.  Here
T_k(H) is computed once ((K-1) SpMMs on `out` channels, written in place into the basis buffer
S = [X | T_0(H) | .. | T_{K-1}(H)]) and ONE GEMM produces all four gate pre-activations; without autograd that GEMM
is the wgmma kernel with the LSTM gate chain in its epilogue (`stmp_gemm_lstm_f32`, zero peepholes -- GCLSTM has
none, and its output gate therefore does not depend on the new cell state, gc_lstm.py:139-145).

Inside the row-split envelope (K <= 2, out_channels 32 or 64, in_channels <= 16, 2-D X; any graph) a step is one launch of the
row-split LSTM cell kernel with the basis [X | H | Op H] and no peepholes, for inference and training alike; training adds its
hand-written backward (ops.lstm_rows_train).  At 64 channels, inference with in_channels % 4 == 0 on graphs of
ops.LSTM_WIDE_ROWS_GEMM_NODES nodes or more keeps the SpMM + wgmma route, which is faster there (DESIGN §4o)."""
import torch

from ... import _lib, ops
from ...plan import _require_cuda
from ._cheb import ChebParams, ChebPlanMixin, broadcast_states, glorot_


class GCLSTM(torch.nn.Module, ChebPlanMixin):
    def __init__(self, in_channels: int, out_channels: int, K: int, normalization: str = "sym", bias: bool = True):
        super().__init__()
        self.in_channels, self.out_channels, self.K = in_channels, out_channels, K
        self.normalization, self.bias = normalization, bias
        P = torch.nn.Parameter
        # creation order mirrors the reference (gc_lstm.py:52-110) so a seeded init consumes the RNG identically:
        # the four ChebConvs draw at construction, the dense W_g afterwards
        for g in "ifco":
            setattr(self, f"conv_{g}", ChebParams(out_channels, out_channels, K, bias))
            setattr(self, f"W_{g}", P(torch.empty(in_channels, out_channels)))
            setattr(self, f"b_{g}", P(torch.empty(1, out_channels)))
        for g in "ifco":
            glorot_(getattr(self, f"W_{g}"))
        for g in "ifco":
            torch.nn.init.zeros_(getattr(self, f"b_{g}"))
        self.register_buffer("_no_peephole", torch.zeros(out_channels), persistent=False)
        self._init_plans()
        self._pack = ops.PackCache()
        self._rows_pack = ops.PackCache()
        self.fused_training = True      # False: op-for-op autograd path (tests compare the two)

    def _weight(self):
        """(in + K*out, 4*out): rows [W_g ; lins[0]^T ; .. ; lins[K-1]^T], gate columns i,f,c,o."""
        cols = []
        for g in "ifco":
            conv = getattr(self, f"conv_{g}")
            cols.append(torch.cat([getattr(self, f"W_{g}")] + [l.weight.t() for l in conv.lins], dim=0))
        return torch.cat(cols, dim=1)

    def _gate_bias(self):
        bs = []
        for g in "ifco":
            b = getattr(self, f"b_{g}").reshape(-1)
            cb = getattr(self, f"conv_{g}").bias
            bs.append(b if cb is None else b + cb)
        return bs

    def _rows_packed(self):
        """(w [4 Co, nb], b [4 Co]) for stmp_lstm_rows_fwd / stmp_lstm_wide_rows_fwd: columns [X | H | Op H] (W_g transposed), b =
        conv_g.bias + b_g (one pack launch per weight update)."""
        def build():
            convs = [getattr(self, f"conv_{g}") for g in "ifco"]
            wx = torch.stack([getattr(self, f"W_{g}") for g in "ifco"])
            wh = torch.stack([torch.stack([c.lins[k].weight for k in range(self.K)]) for c in convs])
            bh = torch.stack([c.bias for c in convs]) if self.bias else None
            bg = torch.cat([getattr(self, f"b_{g}") for g in "ifco"])
            return ops.lstm_rows_pack_weights(_lib.LSTM_GC, self.K - 1, self.in_channels, wx, wh, None, bh, bg)
        return self._rows_pack.get(list(self.parameters()), build)

    def _rows_spec(self):
        """(spec, params) of ops.lstm_rows_train: where each parameter's gradient sits in the packed weight gradient (4 Co, nb) and the
        bias gradient -- the inverse of `_rows_packed`.  W_g (in, out) receives its block transposed; both biases of a gate get the gate's
        block."""
        spec, params = [], []
        Ci, Co = self.in_channels, self.out_channels
        for gi, g in enumerate("ifco"):
            conv = getattr(self, f"conv_{g}")
            spec.append(("wt", Co * gi, Co, 0, Ci))
            params.append(getattr(self, f"W_{g}"))
            for k in range(self.K):
                spec.append(("w", Co * gi, Co, Ci + Co * k, Co))
                params.append(conv.lins[k].weight)
            if conv.bias is not None:
                spec.append(("b", Co * gi, Co))
                params.append(conv.bias)
            spec.append(("b", Co * gi, Co))
            params.append(getattr(self, f"b_{g}"))
        return spec, params

    def _rows_ok(self, plan, X, H, C, training):
        """The row-split route: K <= 2, out_channels 32 or 64, in_channels <= 16, 2-D float32 X, H and C None or (N, out_channels) float32
        (the module's attributes are checked before the library is consulted); training calls also need `fused_training`.  At 64 channels,
        inference that the SpMM + wgmma route serves stays there on large graphs (ops.lstm_rows_for_no_grad)."""
        Co = self.out_channels
        if self.K > 2 or Co not in (32, 64) or self.in_channels > 16 or X.dim() != 2 or X.dtype != torch.float32:
            return False
        if any(S is not None and (S.shape != (X.size(0), Co) or S.dtype != torch.float32) for S in (H, C)):
            return False
        if training and not self.fused_training:
            return False
        if not training and not ops.lstm_rows_for_no_grad(plan, self.in_channels, Co):
            return False
        return ops.lstm_rows_supported(plan, _lib.LSTM_GC, self.K - 1, self.in_channels, Co)

    def forward(self, X: torch.FloatTensor, edge_index: torch.LongTensor, edge_weight: torch.FloatTensor = None,
                H: torch.FloatTensor = None, C: torch.FloatTensor = None, lambda_max: torch.Tensor = None):
        _require_cuda(X, "X")
        N, Ci, Co, K = X.size(-2), self.in_channels, self.out_channels, self.K
        plan = self._cheb_plan(edge_index, edge_weight, N, self.normalization, lambda_max)
        needs_grad = torch.is_grad_enabled() and (any(p.requires_grad for p in self.parameters()) or X.requires_grad
                                                  or (H is not None and H.requires_grad) or (C is not None and C.requires_grad))
        if self._rows_ok(plan, X, H, C, needs_grad):    # the row-split cell kernel (stmp_lstm_rows_*): one launch per step
            w, b = self._rows_packed()
            if needs_grad:
                spec, params = self._rows_spec()
                return ops.lstm_rows_train(plan, _lib.LSTM_GC, K - 1, X, H, C, w, b, None, spec, params)
            return ops.lstm_rows_fwd(plan, _lib.LSTM_GC, K - 1, X, H, C, w, b, None)
        X, (H, C) = broadcast_states(X, (H, C), Co)
        width = Ci + K * Co
        if not needs_grad:
            # the basis is built in place: T_k(H) lands in its column block of S straight from the SpMM kernel
            S = torch.empty(*X.shape[:-1], width, device=X.device, dtype=torch.float32)
            S[..., :Ci] = X
            S[..., Ci:Ci + Co] = H
            for k in range(1, K):
                if k == 1:
                    ops.spmm_cols(plan, 0, S, Ci, Ci + Co, Co)
                else:
                    ops.spmm_cols(plan, 0, S, Ci + (k - 1) * Co, Ci + k * Co, Co, alpha=2.0, z_col=Ci + (k - 2) * Co, beta=-1.0)
            if Co in (32, 64) and width % 4 == 0:
                packed, gb = self._pack.get(list(self.parameters()), lambda: (ops.gemm_prepack(self._weight()), self._gate_bias()))
                z = self._no_peephole
                try:
                    return ops.gemm_lstm(S, packed, width, Co, None, C.contiguous(), z, z, z, gb[0], gb[1], gb[2], gb[3])
                except _lib.StmpUnsupported:
                    pass
            pre = torch.matmul(S, self._weight())
            gb = self._gate_bias()
            pi, pf, pc, po = (pre[..., j * Co:(j + 1) * Co].contiguous() for j in range(4))
            z = self._no_peephole
            Cn = ops.lstm_ifc(pi, pf, pc, C, z, z, gb[0], gb[1], gb[2])
            return ops.lstm_oh(po, Cn, z, gb[3]), Cn
        T = [H]
        if K > 1:
            T.append(ops.spmm(plan, 0, H))
        for _ in range(2, K):
            T.append(ops.spmm(plan, 0, T[-1], alpha=2.0, z=T[-2], beta=-1.0))
        pre = torch.matmul(torch.cat([X] + T, dim=-1), self._weight())
        gb = self._gate_bias()
        pi, pf, pc, po = (pre[..., j * Co:(j + 1) * Co] for j in range(4))
        I = torch.sigmoid(pi + gb[0])
        Fg = torch.sigmoid(pf + gb[1])
        Cn = Fg * C + I * torch.tanh(pc + gb[2])
        O = torch.sigmoid(po + gb[3])
        return O * torch.tanh(Cn), Cn
