"""MPNNLSTM -- drop-in for torch_geometric_temporal/nn/recurrent/mpnn_lstm.py: the reference's constructor and attributes, GCNConv's keys
under `_convolution_{1,2}` (`lin.weight`, `bias`), real torch.nn.BatchNorm1d under `_batch_norm_{1,2}` and torch.nn.LSTM under
`_recurrent_{1,2}`, created in the reference's order, so the state_dict keys and a seeded initialisation equal the reference's.

One call: S = X's skip features (every feature of step 0, the last feature of steps 1 .. window-1), Z1 = dropout(BN1(relu(GCNConv1(X)))),
Z2 = the same of Z1 on the same graph, the two LSTMs over `window` steps of [Z1 | Z2], and H = [h1 | h2 | S].  GCNConv's gcn_norm runs over
X.size(0) nodes (all B * window * num_nodes rows), as PyG's does.  BatchNorm follows each BN module's `training`, dropout the module's.

Calls run on the row-split kernels (DESIGN §4t: stmp_mpnn_rows_fwd, three launches; training calls add a hand-written backward,
stmp_mpnn_rows_bwd + _wgrad) when X is 2-D float32, the parameters and BatchNorm's running statistics are float32 (the statistics
contiguous), edge_weight is None or a float32 (E,) vector that needs no gradient, both BNs are affine with running statistics and in the
same mode, p < 1 and the library supports the shape (hidden_size = 32, in_channels <= 64); training calls also need `fused_training`.
BatchNorm's running statistics and num_batches_tracked are updated on the device in training mode, under no_grad too.  Everything else
runs op for op on the GPU (ops.spmm on the plan in float32, index_add on gcn_norm otherwise, and the module's own BN and LSTM modules).

Dropout: in training mode with p > 0 both routes draw u = torch.rand(2, R, 32) on X's device and keep an element where u >= p, scaling
it by 1 / (1 - p).  The masks are equal in distribution to F.dropout's but are not the same draw of the random stream: the one intended
difference from the reference."""
import torch

from ... import _lib, ops
from ...plan import PlanCache, _require_cuda
from .evolvegcn import gcn_norm
from .temporalgcn import GCNParams


class MPNNLSTM(torch.nn.Module):
    def __init__(self, in_channels: int, hidden_size: int, num_nodes: int, window: int, dropout: float):
        super().__init__()
        self.window = window
        self.num_nodes = num_nodes
        self.hidden_size = hidden_size
        self.dropout = dropout
        self.in_channels = in_channels
        self._create_parameters_and_layers()
        self._plans = PlanCache()
        self.fused_training = True      # False: op-for-op autograd path for training calls (tests compare the two)

    def _create_parameters_and_layers(self):
        self._convolution_1 = GCNParams(self.in_channels, self.hidden_size)
        self._convolution_2 = GCNParams(self.hidden_size, self.hidden_size)
        self._batch_norm_1 = torch.nn.BatchNorm1d(self.hidden_size)
        self._batch_norm_2 = torch.nn.BatchNorm1d(self.hidden_size)
        self._recurrent_1 = torch.nn.LSTM(2 * self.hidden_size, self.hidden_size, 1)
        self._recurrent_2 = torch.nn.LSTM(self.hidden_size, self.hidden_size, 1)

    def _plan(self, edge_index, edge_weight, num_nodes):
        """gcn_norm's operator with remaining self loops of fill 1 over all rows, shared by both convolutions."""
        return self._plans.get(_lib.FLAVOR_GCN, edge_index, edge_weight, num_nodes, flags=0)

    def _uniforms(self, R, device):
        """The dropout uniforms of one training call: (2, R, hidden_size), one layer each."""
        return torch.rand(2, R, self.hidden_size, device=device)

    def _fused_ok(self, X, edge_weight, needs_grad):
        """The module's conditions for the row-split kernels (the library decides the widths: stmp_mpnn_rows_supported)."""
        if (needs_grad and not self.fused_training) or X.dim() != 2 or X.dtype != torch.float32 or X.size(1) != self.in_channels:
            return False
        if any(p.dtype != torch.float32 for p in self.parameters()):
            return False
        if edge_weight is not None and (edge_weight.dtype != torch.float32 or edge_weight.dim() != 1 or edge_weight.requires_grad):
            return False
        bn1, bn2 = self._batch_norm_1, self._batch_norm_2
        if not all(bn.affine and bn.track_running_stats for bn in (bn1, bn2)) or bn1.training != bn2.training:
            return False
        if any(t.dtype != torch.float32 or not t.is_contiguous() for bn in (bn1, bn2) for t in (bn.running_mean, bn.running_var)):
            return False
        return self.dropout < 1

    def _conv(self, conv, X, plan, edge_index, edge_weight):
        """GCNConv op for op: Op (X W^T) + b."""
        XW = torch.matmul(X, conv.lin.weight.t())
        if XW.dtype == torch.float32 and (edge_weight is None or not edge_weight.requires_grad):
            return ops.spmm(plan(), 0, XW) + conv.bias
        ei, ew = gcn_norm(edge_index, edge_weight, X.size(0), dtype=XW.dtype)
        msg = ew.view(-1, 1).to(XW.dtype) * XW.index_select(0, ei[0])
        return XW.new_zeros(XW.shape).index_add(0, ei[1], msg) + conv.bias

    def forward(self, X: torch.FloatTensor, edge_index: torch.LongTensor, edge_weight: torch.FloatTensor) -> torch.FloatTensor:
        T, N, F = self.window, self.num_nodes, self.in_channels
        S4 = X.view(-1, T, N, F)             # the reference's shape error, before any launch
        R = X.size(0)
        for bn in (self._batch_norm_1, self._batch_norm_2):
            if bn.training and R == 1:
                raise ValueError(f"Expected more than 1 value per channel when training, got input size {torch.Size([1, self.hidden_size])}")
        _require_cuda(X, "X")
        p = float(self.dropout)
        u = self._uniforms(R, X.device) if self.training and p > 0 else None
        needs_grad = torch.is_grad_enabled() and (X.requires_grad or any(q.requires_grad for q in self.parameters()))
        plan = lambda: self._plan(edge_index, edge_weight, R)
        if self._fused_ok(X, edge_weight, needs_grad) and ops.mpnn_rows_supported(plan(), F, self.hidden_size, T):
            args = (plan(), X, N, T, self._convolution_1, self._convolution_2, self._batch_norm_1, self._batch_norm_2, self._recurrent_1,
                    self._recurrent_2, self._batch_norm_1.training, p if u is not None else 0.0, u)
            return ops.mpnn_rows_train(*args) if needs_grad else ops.mpnn_rows_fwd(*args)
        S = S4.transpose(1, 2).reshape(-1, T, F)
        S = torch.cat([S[:, 0, :]] + [S[:, t, F - 1].unsqueeze(1) for t in range(1, T)], dim=1)
        Z = []
        for layer, (conv, bn) in enumerate(((self._convolution_1, self._batch_norm_1), (self._convolution_2, self._batch_norm_2))):
            Y = bn(torch.relu(self._conv(conv, Z[-1] if Z else X, plan, edge_index, edge_weight)))
            if u is not None:
                Y = Y * ((u[layer] >= p).to(Y.dtype) / (1 - p)) if p < 1 else Y * 0
            Z.append(Y)
        H = torch.cat(Z, dim=1)
        H = H.view(-1, T, N, H.size(1)).transpose(0, 1).contiguous().view(T, -1, H.size(1))
        H, (H_1, _) = self._recurrent_1(H)
        H, (H_2, _) = self._recurrent_2(H)
        return torch.cat([H_1[0], H_2[0], S], dim=1)
