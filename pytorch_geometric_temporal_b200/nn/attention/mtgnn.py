"""MTGNN -- drop-in for torch_geometric_temporal/nn/attention/mtgnn.py: the reference's constructors, attributes, submodule order and
initialisation (every `_reset_parameters` re-draws all parameters: xavier_uniform_ for dim > 1, uniform_ otherwise, so the 3-D
LayerNorm weights and the embeddings are xavier-initialised), so the state_dict keys and a seeded initialisation equal the reference's.

Reference behaviour kept as it is: `_idx` is a plain attribute, not a buffer; the input is left-padded when seq_length is below the
receptive field; DilatedInception gives each branch int(c_out / len(kernel_set)) channels and cuts every branch to the last branch's
length; LayerNormalization indexes its affine parameters with idx; with FE, nodevec2 is nodevec1 (and FE.shape[1] is asserted);
MixProp stores `dropout` and never applies it; a predefined A_tilde is not permuted by idx; a layer adds MixProp(X, A) and
MixProp(X, A^T); the output is (B, out_dim, N, 1).

Every convolution runs as an fp32 contraction (`_conv`: unfold + einsum on cuBLAS), because cuDNN would use TF32 in forward and
backward.  The graph work runs on the fused kernels (DESIGN §4x, mtgnn.cu) when the model's graph is learned, or predefined and not
requiring grad, X is CUDA float32 and the shapes are inside stmp_mtgnn_supported (N <= 4096, k <= 64, node_dim <= 64, conv_channels
<= 64, gcn_depth 1..4); a training call also needs `fused_training`.  The top-k graph of GraphConstructor is then built once per call
as sparse operators, and each layer's two MixProps run as hop chains over them.  Everything else (float64, gcn_true=False, larger
graphs, A_tilde requiring grad, fused_training = False) runs op for op on the GPU as the reference's algebra, and so does a graph
whose node count differs from X's (the reference's einsum then raises its size error; the kernels never see such a graph).  Dropout stays as
F.dropout at the reference's call sites, so both routes draw the same masks from the same generator state."""
from typing import NamedTuple, Optional

import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.nn import init

from ... import ops
from ...plan import _require_cuda
from .astgcn import _conv_1xk


def _reset(module: nn.Module):
    for p in module.parameters():
        if p.dim() > 1:
            nn.init.xavier_uniform_(p)
        else:
            nn.init.uniform_(p)


def _conv(conv: nn.Conv2d, x: torch.Tensor) -> torch.Tensor:
    """An MTGNN Conv2d (kernel (1, k), stride 1, no padding, dilation (1, d)) on (B, C, N, T) as an fp32 contraction."""
    d = conv.dilation[1]
    if d == 1:
        return _conv_1xk(conv, x)
    k = conv.kernel_size[1]
    taps = x.unfold(-1, (k - 1) * d + 1, 1)[..., ::d]            # (B, C, N, T_out, k): the dilated taps of each output step
    out = torch.einsum("bcntk,ock->bont", taps, conv.weight[:, :, 0, :])
    return out if conv.bias is None else out + conv.bias.view(1, -1, 1, 1)


class _Graph(NamedTuple):
    """A graph on the fused kernels: the operator values and the pattern of stmp_mtgnn_* (include/stmp.h), N nodes, row width w."""
    vals: torch.Tensor
    pattern: torch.Tensor
    n: int
    w: int


class _DenseGraphCache:
    """Sparse structures of a predefined A_tilde, keyed on the tensor's (data_ptr, _version, shape, device)."""

    def __init__(self):
        self._key, self._graph = None, None

    def get(self, A: torch.Tensor) -> _Graph:
        key = (A.data_ptr(), A._version, tuple(A.shape), str(A.device))
        if key != self._key:
            pattern, _, vals, w = ops.mtgnn_graph_dense(A)
            self._key, self._graph = key, _Graph(vals, pattern, A.shape[0], w)
        return self._graph


class Linear(nn.Module):
    def __init__(self, c_in: int, c_out: int, bias: bool = True):
        super().__init__()
        self._mlp = torch.nn.Conv2d(c_in, c_out, kernel_size=(1, 1), padding=(0, 0), stride=(1, 1), bias=bias)
        self._reset_parameters()

    def _reset_parameters(self):
        _reset(self)

    def forward(self, X: torch.FloatTensor) -> torch.FloatTensor:
        return _conv(self._mlp, X)


class MixProp(nn.Module):
    """Mix-hop propagation over a dense A, op for op: H_k = alpha X + (1 - alpha) A~ H_{k-1}, A~ = (A + I) / rowsum(A + I), then the
    MLP over [H_0 | ... | H_gdep].  Inside MTGNN a layer's two MixProps run on the fused kernels instead (ops.mtgnn_mixprop)."""

    def __init__(self, c_in: int, c_out: int, gdep: int, dropout: float, alpha: float):
        super().__init__()
        self._mlp = Linear((gdep + 1) * c_in, c_out)
        self._gdep = gdep
        self._dropout = dropout
        self._alpha = alpha
        self._reset_parameters()

    def _reset_parameters(self):
        _reset(self)

    def forward(self, X: torch.FloatTensor, A: torch.FloatTensor) -> torch.FloatTensor:
        _require_cuda(X, "X")
        A = A + torch.eye(A.size(0), device=X.device, dtype=A.dtype)
        A = A / A.sum(1).view(-1, 1)
        H, hops = X, [X]
        for _ in range(self._gdep):
            H = self._alpha * X + (1 - self._alpha) * torch.einsum("ncwl,vw->ncvl", (H, A))
            hops.append(H)
        return self._mlp(torch.cat(hops, dim=1))


class DilatedInception(nn.Module):
    def __init__(self, c_in: int, c_out: int, kernel_set: list, dilation_factor: int):
        super().__init__()
        self._time_conv = nn.ModuleList()
        self._kernel_set = kernel_set
        per_branch = int(c_out / len(self._kernel_set))
        for kern in self._kernel_set:
            self._time_conv.append(nn.Conv2d(c_in, per_branch, (1, kern), dilation=(1, dilation_factor)))
        self._reset_parameters()

    def _reset_parameters(self):
        _reset(self)

    def forward(self, X_in: torch.FloatTensor) -> torch.FloatTensor:
        branches = [_conv(conv, X_in) for conv in self._time_conv]
        T = branches[-1].size(3)
        return torch.cat([b[..., -T:] for b in branches], dim=1)


class GraphConstructor(nn.Module):
    def __init__(self, nnodes: int, k: int, dim: int, alpha: float, xd: Optional[int] = None):
        super().__init__()
        if xd is not None:
            self._static_feature_dim = xd
            self._linear1 = nn.Linear(xd, dim)
            self._linear2 = nn.Linear(xd, dim)
        else:
            self._embedding1 = nn.Embedding(nnodes, dim)
            self._embedding2 = nn.Embedding(nnodes, dim)
            self._linear1 = nn.Linear(dim, dim)
            self._linear2 = nn.Linear(dim, dim)
        self._k = k
        self._alpha = alpha
        self._reset_parameters()

    def _reset_parameters(self):
        _reset(self)

    def node_vectors(self, idx: torch.LongTensor, FE: Optional[torch.FloatTensor] = None):
        """M1 = tanh(alpha linear1(nodevec1)), M2 = tanh(alpha linear2(nodevec2)), each (len(idx), dim)."""
        if FE is None:
            nodevec1 = self._embedding1(idx)
            nodevec2 = self._embedding2(idx)
        else:
            assert FE.shape[1] == self._static_feature_dim
            nodevec1 = FE[idx, :]
            nodevec2 = nodevec1
        return torch.tanh(self._alpha * self._linear1(nodevec1)), torch.tanh(self._alpha * self._linear2(nodevec2))

    def forward(self, idx: torch.LongTensor, FE: Optional[torch.FloatTensor] = None) -> torch.FloatTensor:
        """The dense adjacency: relu(tanh(alpha (M1 M2^T - M2 M1^T))) with the k largest entries of each row kept."""
        m1, m2 = self.node_vectors(idx, FE)
        a = torch.mm(m1, m2.transpose(1, 0)) - torch.mm(m2, m1.transpose(1, 0))
        A = F.relu(torch.tanh(self._alpha * a))
        mask = torch.zeros(idx.size(0), idx.size(0), device=A.device)
        _, cols = A.topk(self._k, 1)
        mask.scatter_(1, cols, 1.0)
        return A * mask

    def sparse(self, idx: torch.LongTensor, FE: Optional[torch.FloatTensor], train: bool) -> _Graph:
        """The same graph as sparse operators on the fused kernels (stmp_mtgnn_graph_fwd); differentiable with `train`."""
        n = idx.size(0)
        if self._k > n:
            raise RuntimeError("selected index k out of range")
        m1, m2 = self.node_vectors(idx, FE)
        vals, pattern = ops.mtgnn_graph(m1, m2, self._k, float(self._alpha), train)
        return _Graph(vals, pattern, n, self._k)


class LayerNormalization(nn.Module):
    __constants__ = ["normalized_shape", "weight", "bias", "eps", "elementwise_affine"]

    def __init__(self, normalized_shape: int, eps: float = 1e-5, elementwise_affine: bool = True):
        super().__init__()
        self._normalized_shape = tuple(normalized_shape)
        self._eps = eps
        self._elementwise_affine = elementwise_affine
        if self._elementwise_affine:
            self._weight = nn.Parameter(torch.Tensor(*normalized_shape))
            self._bias = nn.Parameter(torch.Tensor(*normalized_shape))
        else:
            self.register_parameter("_weight", None)
            self.register_parameter("_bias", None)
        self._reset_parameters()

    def _reset_parameters(self):
        if self._elementwise_affine:
            init.ones_(self._weight)
            init.zeros_(self._bias)

    def forward(self, X: torch.FloatTensor, idx: torch.LongTensor) -> torch.FloatTensor:
        if self._elementwise_affine:
            return F.layer_norm(X, tuple(X.shape[1:]), self._weight[:, idx, :], self._bias[:, idx, :], self._eps)
        return F.layer_norm(X, tuple(X.shape[1:]), self._weight, self._bias, self._eps)


class MTGNNLayer(nn.Module):
    def __init__(self, dilation_exponential: int, rf_size_i: int, kernel_size: int, j: int, residual_channels: int,
                 conv_channels: int, skip_channels: int, kernel_set: list, new_dilation: int, layer_norm_affline: bool,
                 gcn_true: bool, seq_length: int, receptive_field: int, dropout: float, gcn_depth: int, num_nodes: int,
                 propalpha: float):
        super().__init__()
        self._dropout = dropout
        self._gcn_true = gcn_true
        if dilation_exponential > 1:
            rf_size_j = int(rf_size_i + (kernel_size - 1) * (dilation_exponential ** j - 1) / (dilation_exponential - 1))
        else:
            rf_size_j = rf_size_i + j * (kernel_size - 1)
        self._filter_conv = DilatedInception(residual_channels, conv_channels, kernel_set=kernel_set, dilation_factor=new_dilation)
        self._gate_conv = DilatedInception(residual_channels, conv_channels, kernel_set=kernel_set, dilation_factor=new_dilation)
        self._residual_conv = nn.Conv2d(in_channels=conv_channels, out_channels=residual_channels, kernel_size=(1, 1))
        span = max(seq_length, receptive_field) - rf_size_j + 1
        self._skip_conv = nn.Conv2d(in_channels=conv_channels, out_channels=skip_channels, kernel_size=(1, span))
        if gcn_true:
            self._mixprop_conv1 = MixProp(conv_channels, residual_channels, gcn_depth, dropout, propalpha)
            self._mixprop_conv2 = MixProp(conv_channels, residual_channels, gcn_depth, dropout, propalpha)
        self._normalization = LayerNormalization((residual_channels, num_nodes, span), elementwise_affine=layer_norm_affline)
        self._reset_parameters()

    def _reset_parameters(self):
        _reset(self)

    def forward(self, X: torch.FloatTensor, X_skip: torch.FloatTensor, A_tilde, idx: torch.LongTensor, training: bool):
        """A_tilde: a dense (N, N) adjacency, or the model's graph on the fused kernels."""
        X_residual = X
        X = torch.tanh(self._filter_conv(X)) * torch.sigmoid(self._gate_conv(X))
        X = F.dropout(X, self._dropout, training=training)
        X_skip = _conv(self._skip_conv, X) + X_skip
        if self._gcn_true:
            if isinstance(A_tilde, _Graph):
                if X.shape[2] != A_tilde.n:
                    raise RuntimeError(f"einsum(): subscript w has size {A_tilde.n} for operand 1 which does not broadcast with "
                                       f"previously seen size {X.shape[2]}: the graph has {A_tilde.n} nodes, X has {X.shape[2]}")
                m1, m2 = self._mixprop_conv1, self._mixprop_conv2
                train = torch.is_grad_enabled() and (X.requires_grad or A_tilde.vals.requires_grad or
                                                     any(p.requires_grad for p in (m1._mlp._mlp.weight, m2._mlp._mlp.weight)))
                X = ops.mtgnn_mixprop(X, A_tilde.vals, A_tilde.pattern, A_tilde.w, m1._gdep, float(m1._alpha), m1._mlp._mlp.weight,
                                      m1._mlp._mlp.bias, m2._mlp._mlp.weight, m2._mlp._mlp.bias, train)
            else:
                X = self._mixprop_conv1(X, A_tilde) + self._mixprop_conv2(X, A_tilde.transpose(1, 0))
        else:
            X = _conv(self._residual_conv, X)
        X = X + X_residual[:, :, :, -X.size(3):]
        X = self._normalization(X, idx)
        return X, X_skip


def fused_route(dtype, is_cuda: bool, n: int, k: int, dim: int, channels: int, depth: int, batch: int, steps: int,
                gcn_true: bool, needs_grad: bool, fused_training: bool) -> bool:
    """Whether an MTGNN call runs its graph work on the fused kernels (the library decides the envelope: stmp_mtgnn_supported)."""
    if not gcn_true or dtype != torch.float32 or not is_cuda or (needs_grad and not fused_training):
        return False
    return ops.mtgnn_supported(n, k, dim, channels, depth, batch, steps)


class MTGNN(nn.Module):
    def __init__(self, gcn_true: bool, build_adj: bool, gcn_depth: int, num_nodes: int, kernel_set: list, kernel_size: int,
                 dropout: float, subgraph_size: int, node_dim: int, dilation_exponential: int, conv_channels: int,
                 residual_channels: int, skip_channels: int, end_channels: int, seq_length: int, in_dim: int, out_dim: int,
                 layers: int, propalpha: float, tanhalpha: float, layer_norm_affline: bool, xd: Optional[int] = None):
        super().__init__()
        self._gcn_true = gcn_true
        self._build_adj_true = build_adj
        self._num_nodes = num_nodes
        self._dropout = dropout
        self._seq_length = seq_length
        self._layers = layers
        self._idx = torch.arange(self._num_nodes)
        self._mtgnn_layers = nn.ModuleList()
        self._graph_constructor = GraphConstructor(num_nodes, subgraph_size, node_dim, alpha=tanhalpha, xd=xd)
        self._set_receptive_field(dilation_exponential, kernel_size, layers)
        new_dilation = 1
        for j in range(1, layers + 1):
            self._mtgnn_layers.append(MTGNNLayer(
                dilation_exponential=dilation_exponential, rf_size_i=1, kernel_size=kernel_size, j=j,
                residual_channels=residual_channels, conv_channels=conv_channels, skip_channels=skip_channels, kernel_set=kernel_set,
                new_dilation=new_dilation, layer_norm_affline=layer_norm_affline, gcn_true=gcn_true, seq_length=seq_length,
                receptive_field=self._receptive_field, dropout=dropout, gcn_depth=gcn_depth, num_nodes=num_nodes,
                propalpha=propalpha))
            new_dilation *= dilation_exponential
        self._setup_conv(in_dim, skip_channels, end_channels, residual_channels, out_dim)
        self._reset_parameters()
        self._gcn_depth, self._conv_channels, self._node_dim = gcn_depth, conv_channels, node_dim
        self.fused_training = True
        self._dense_cache = _DenseGraphCache()
        self._idx_on = {}

    def _device_idx(self, device) -> torch.Tensor:
        """`_idx` on the input's device, copied once (a copy per call would stop a CUDA-graph capture)."""
        key = (str(device), self._idx.data_ptr())
        if key not in self._idx_on:
            self._idx_on = {key: self._idx.to(device)}
        return self._idx_on[key]

    def _setup_conv(self, in_dim, skip_channels, end_channels, residual_channels, out_dim):
        self._start_conv = nn.Conv2d(in_channels=in_dim, out_channels=residual_channels, kernel_size=(1, 1))
        long_input = self._seq_length > self._receptive_field
        self._skip_conv_0 = nn.Conv2d(in_channels=in_dim, out_channels=skip_channels,
                                      kernel_size=(1, self._seq_length if long_input else self._receptive_field), bias=True)
        self._skip_conv_E = nn.Conv2d(in_channels=residual_channels, out_channels=skip_channels,
                                      kernel_size=(1, self._seq_length - self._receptive_field + 1 if long_input else 1), bias=True)
        self._end_conv_1 = nn.Conv2d(in_channels=skip_channels, out_channels=end_channels, kernel_size=(1, 1), bias=True)
        self._end_conv_2 = nn.Conv2d(in_channels=end_channels, out_channels=out_dim, kernel_size=(1, 1), bias=True)

    def _reset_parameters(self):
        _reset(self)

    def _set_receptive_field(self, dilation_exponential, kernel_size, layers):
        if dilation_exponential > 1:
            self._receptive_field = int(1 + (kernel_size - 1) * (dilation_exponential ** layers - 1) / (dilation_exponential - 1))
        else:
            self._receptive_field = layers * (kernel_size - 1) + 1

    def _fused(self, X_in: torch.Tensor, n: int, width: int, dim: int) -> bool:
        """Whether this call's graph work runs fused: a graph of n nodes and row width `width`, built from node vectors of width dim
        (1 for a predefined graph, which has none).  A graph whose node count differs from X's runs op for op, where the reference's
        einsum raises its size error before any kernel of this library launches."""
        if n != X_in.shape[2]:
            return False
        needs_grad = torch.is_grad_enabled() and (X_in.requires_grad or any(p.requires_grad for p in self.parameters()))
        steps = max(self._seq_length, self._receptive_field)
        return fused_route(X_in.dtype, X_in.is_cuda, n, width, dim, self._conv_channels, self._gcn_depth, X_in.shape[0],
                           steps, self._gcn_true, needs_grad, self.fused_training)

    def _graph(self, X_in, A_tilde, idx, FE):
        """The layers' adjacency: a dense tensor (op for op) or a _Graph on the fused kernels."""
        if not self._gcn_true:
            return A_tilde
        if self._build_adj_true:
            ids = self._device_idx(X_in.device) if idx is None else idx
            gc = self._graph_constructor
            if self._fused(X_in, ids.size(0), min(gc._k, ids.size(0)), self._node_dim):
                train = torch.is_grad_enabled() and (any(p.requires_grad for p in gc.parameters()) or
                                                     (FE is not None and FE.requires_grad))
                return gc.sparse(ids, FE, train)
            return gc(ids, FE=FE)
        if A_tilde is not None and not (A_tilde.requires_grad and torch.is_grad_enabled()) and A_tilde.dim() == 2 and \
                A_tilde.shape[0] == A_tilde.shape[1] and A_tilde.dtype == torch.float32 and A_tilde.is_cuda and \
                self._fused(X_in, A_tilde.shape[0], 1, 1):
            return self._dense_cache.get(A_tilde)
        return A_tilde

    def forward(self, X_in: torch.FloatTensor, A_tilde: Optional[torch.FloatTensor] = None, idx: Optional[torch.LongTensor] = None,
                FE: Optional[torch.FloatTensor] = None) -> torch.FloatTensor:
        _require_cuda(X_in, "X_in")
        seq_len = X_in.size(3)
        assert seq_len == self._seq_length, "Input sequence length not equal to preset sequence length."
        if self._seq_length < self._receptive_field:
            X_in = nn.functional.pad(X_in, (self._receptive_field - self._seq_length, 0, 0, 0))
        A_tilde = self._graph(X_in, A_tilde, idx, FE)
        X = _conv(self._start_conv, X_in)
        X_skip = _conv(self._skip_conv_0, F.dropout(X_in, self._dropout, training=self.training))
        ids = self._device_idx(X_in.device) if idx is None else idx
        for mtgnn in self._mtgnn_layers:
            X, X_skip = mtgnn(X, X_skip, A_tilde, ids, self.training)
        X_skip = _conv(self._skip_conv_E, X) + X_skip
        X = F.relu(X_skip)
        X = F.relu(_conv(self._end_conv_1, X))
        return _conv(self._end_conv_2, X)
