"""DyGrEncoder -- drop-in for torch_geometric_temporal/nn/recurrent/dygrae.py: constructor `(conv_out_channels, conv_num_layers,
conv_aggr, lstm_out_channels, lstm_num_layers)`, `forward(X, edge_index, edge_weight=None, H=None, C=None) -> (H_tilde, H, C)`, submodules
`conv_layer` (PyG GatedGraphConv's parameters `weight`, `rnn.*`) and `recurrent_layer` (a torch.nn.LSTM), so the state_dict keys and a
seeded initialisation equal the reference's.

GatedGraphConv runs on the row-split kernels (stmp_ggc_rows_*, DESIGN §4r) for 2-D float32 X with in_channels <= C <= 32, as many
layers as the library supports (1 024; _conv_route asks ops.ggc_rows_supported), any aggregation and edge_weight None or a constant
float32 (E,) vector: one launch per layer (one more for max), with a hand-written backward.  The LSTM on top of it is the row-split LSTM
cell on the basis [x | H] (stmp_lstm_rows_*, n_ops = 0) when C <= 16, lstm_out_channels is 32 or 64 and lstm_num_layers is 1; otherwise
the convolution's output goes to the module's own torch.nn.LSTM.  Everything else -- wider or non-float32 inputs, more layers, batched
X, or `fused_training = False` for a training call -- runs op for op on the GPU
(ops.spmm for add and mean in float32, index_select + scatter_reduce "amax" for max and index_add for other dtypes, then the GRUCell and
the LSTM modules)."""
import math

import torch

from ... import _lib, ops
from ...plan import GatedPlan, _require_cuda


class GatedGraphConv(torch.nn.Module):
    """PyG 2.x GatedGraphConv(out_channels, num_layers, aggr, bias): `weight` (num_layers, C, C) registered before `rnn` =
    torch.nn.GRUCell(C, C, bias); reset_parameters draws weight ~ U(-1/sqrt(C), 1/sqrt(C)) after the GRUCell constructor's draws and then
    resets the GRUCell again, in PyG's order."""

    def __init__(self, out_channels: int, num_layers: int, aggr: str = "add", bias: bool = True):
        super().__init__()
        self.out_channels, self.num_layers, self.aggr = out_channels, num_layers, aggr
        self.weight = torch.nn.Parameter(torch.empty(num_layers, out_channels, out_channels))
        self.rnn = torch.nn.GRUCell(out_channels, out_channels, bias=bias)
        self.reset_parameters()

    def reset_parameters(self):
        bound = 1.0 / math.sqrt(self.out_channels)
        with torch.no_grad():
            self.weight.uniform_(-bound, bound)
        self.rnn.reset_parameters()


class DyGrEncoder(torch.nn.Module):
    def __init__(self, conv_out_channels: int, conv_num_layers: int, conv_aggr: str, lstm_out_channels: int, lstm_num_layers: int):
        super().__init__()
        assert conv_aggr in ["mean", "add", "max"], "Wrong aggregator."
        self.conv_out_channels, self.conv_num_layers, self.conv_aggr = conv_out_channels, conv_num_layers, conv_aggr
        self.lstm_out_channels, self.lstm_num_layers = lstm_out_channels, lstm_num_layers
        self.conv_layer = GatedGraphConv(conv_out_channels, conv_num_layers, conv_aggr, bias=True)
        self.recurrent_layer = torch.nn.LSTM(conv_out_channels, lstm_out_channels, lstm_num_layers)
        self._plans = {}
        self._lstm_pack = ops.PackCache()
        self.fused_training = True      # False: op-for-op autograd path for training calls (tests compare the two)

    def _plan(self, edge_index, edge_weight, num_nodes):
        """The gated plan, cached on (data_ptr, _version, shape) of edge_index and edge_weight and the aggregation: no device sync on a
        hit."""
        tk = lambda t: None if t is None else (t.data_ptr(), t._version, tuple(t.shape), t.dtype, t.device)
        key = (tk(edge_index), tk(edge_weight), int(num_nodes), self.conv_aggr)
        hit = self._plans.get(key)
        if hit is not None:
            return hit[0]
        plan = GatedPlan(edge_index, edge_weight, num_nodes, self.conv_aggr)
        if len(self._plans) >= 4:
            self._plans.pop(next(iter(self._plans)))
        self._plans[key] = (plan, edge_index, edge_weight)    # the keyed tensors stay alive, so their addresses are not recycled
        return plan

    def _conv_ok(self, X, edge_weight, training):
        """The module's own conditions for the row-split GatedGraphConv: 2-D float32 X with 1 <= in_channels <= C <= 32, float32
        parameters, edge_weight None or a float32 (E,) vector that needs no gradient; training calls also need `fused_training`."""
        C = self.conv_out_channels
        if X.dim() != 2 or X.dtype != torch.float32 or not 1 <= X.size(1) <= C <= 32 or X.size(0) < 1:
            return False
        if any(p.dtype != torch.float32 for p in self.conv_layer.parameters()):
            return False
        if edge_weight is not None and (edge_weight.dtype != torch.float32 or edge_weight.dim() != 1 or edge_weight.requires_grad):
            return False
        return not (training and not self.fused_training)

    def _conv_route(self, plan, X, edge_weight, training):
        """Whether the convolution runs on the row-split kernels: the module's conditions (_conv_ok), then the library's envelope for this
        plan, layer count and width (ops.ggc_rows_supported: 1 024 layers at most), which is asked and never restated here."""
        if not self._conv_ok(X, edge_weight, training):
            return False
        return ops.ggc_rows_supported(plan, self.conv_num_layers, X.size(1), self.conv_out_channels)

    def _lstm_ok(self, plan, N, H, C):
        """The row-split LSTM stage after a row-split convolution: C <= 16, lstm_out_channels 32 or 64, one LSTM layer, float32 LSTM
        parameters, H and C None or (N, lstm_out_channels) float32."""
        Ho = self.lstm_out_channels
        if self.conv_out_channels > 16 or Ho not in (32, 64) or self.lstm_num_layers != 1:
            return False
        if any(p.dtype != torch.float32 for p in self.recurrent_layer.parameters()):
            return False
        if any(S is not None and (S.shape != (N, Ho) or S.dtype != torch.float32) for S in (H, C)):
            return False
        return ops.lstm_rows_supported(plan, _lib.LSTM_GCONV, 0, self.conv_out_channels, Ho)

    def _lstm_packed(self):
        """(w [4 Ho, C + Ho], b [4 Ho]) of stmp_lstm_rows_fwd on the basis [x | H]: w = [weight_ih_l0 | weight_hh_l0] (gate order i | f | g | o
        is the cell's), b = bias_ih_l0 + bias_hh_l0.  One pack launch per parameter change."""
        r = self.recurrent_layer
        Ho, C = self.lstm_out_channels, self.conv_out_channels

        def build():
            return ops.lstm_rows_pack_weights(_lib.LSTM_GCONV, 0, C, r.weight_ih_l0.view(4, 1, Ho, C), r.weight_hh_l0.view(4, 1, Ho, Ho),
                                              r.bias_ih_l0.view(4, Ho), r.bias_hh_l0.view(4, Ho), torch.zeros(4, Ho, device=r.bias_ih_l0.device))
        return self._lstm_pack.get(list(r.parameters()), build)

    def _lstm_spec(self):
        """(spec, params) of ops.lstm_rows_train: weight_ih_l0 and weight_hh_l0 are the packed gradient's column blocks as they stand, both
        biases the summed bias gradient."""
        r = self.recurrent_layer
        Ho, C = self.lstm_out_channels, self.conv_out_channels
        spec = [("w", 0, 4 * Ho, 0, C), ("w", 0, 4 * Ho, C, Ho), ("b", 0, 4 * Ho), ("b", 0, 4 * Ho)]
        return spec, [r.weight_ih_l0, r.weight_hh_l0, r.bias_ih_l0, r.bias_hh_l0]

    def _conv_op_for_op(self, plan, X, edge_index, edge_weight):
        """PyG GatedGraphConv.forward op for op on the GPU: pad, then per layer m = x W_l, the aggregation, x = GRUCell(m, x)."""
        conv, C = self.conv_layer, self.conv_out_channels
        x = X
        if x.size(-1) < C:
            zero = x.new_zeros(x.size(0), C - x.size(-1))
            x = torch.cat([x, zero], dim=1)
        src, dst = edge_index[0], edge_index[1]
        for i in range(self.conv_num_layers):
            m = torch.matmul(x, conv.weight[i])
            if self.conv_aggr != "max" and m.dtype == torch.float32:
                m = ops.spmm(plan, 0, m)                # the plan's values: w_e, or w_e / cnt(dst) for mean
            else:
                msg = m.index_select(-2, src)
                if edge_weight is not None:
                    msg = edge_weight.view(-1, 1).to(m.dtype) * msg
                if self.conv_aggr == "max":
                    m = m.new_zeros(m.shape).scatter_reduce(0, dst.view(-1, 1).expand_as(msg), msg, "amax", include_self=False)
                else:
                    m = m.new_zeros(m.shape).index_add(0, dst, msg)
                    if self.conv_aggr == "mean":
                        cnt = m.new_zeros(m.size(0)).index_add(0, dst, torch.ones_like(dst, dtype=m.dtype))
                        m = m / cnt.clamp(min=1).unsqueeze(1)
            x = conv.rnn(m, x)
        return x

    def forward(self, X: torch.FloatTensor, edge_index: torch.LongTensor, edge_weight: torch.FloatTensor = None,
                H: torch.FloatTensor = None, C: torch.FloatTensor = None):
        if X.size(-1) > self.conv_out_channels:
            raise ValueError("The number of input channels is not allowed to be larger than the number of output channels")
        if (H is None) != (C is None):
            raise ValueError("Invalid hidden state and cell matrices.")
        _require_cuda(X, "X")
        N = X.size(-2)
        plan = self._plan(edge_index, edge_weight, N)
        params = list(self.parameters())
        needs_grad = torch.is_grad_enabled() and (any(p.requires_grad for p in params) or X.requires_grad
                                                  or (H is not None and H.requires_grad) or (C is not None and C.requires_grad))
        if not self._conv_route(plan, X, edge_weight, needs_grad):
            Ht = self._conv_op_for_op(plan, X, edge_index, edge_weight)
        else:
            g = self.conv_layer
            args = (plan, X, g.weight, g.rnn.weight_ih, g.rnn.weight_hh, g.rnn.bias_ih, g.rnn.bias_hh)
            Ht = ops.ggc_rows_train(*args) if needs_grad else ops.ggc_rows_fwd(*args)
            if self._lstm_ok(plan, N, H, C):          # the row-split LSTM cell on [x | H]: one launch
                w, b = self._lstm_packed()
                if needs_grad:
                    spec, lp = self._lstm_spec()
                    h, c = ops.lstm_rows_train(plan, _lib.LSTM_GCONV, 0, Ht, H, C, w, b, None, spec, lp)
                else:
                    h, c = ops.lstm_rows_fwd(plan, _lib.LSTM_GCONV, 0, Ht, H, C, w, b, None)
                return h.squeeze(), h.clone().squeeze(), c.squeeze()
        Ht = Ht[None, :, :]
        if H is None and C is None:
            Ht, (H, C) = self.recurrent_layer(Ht)
        else:
            Ht, (H, C) = self.recurrent_layer(Ht, (H[None, :, :], C[None, :, :]))
        return Ht.squeeze(), H.squeeze(), C.squeeze()
