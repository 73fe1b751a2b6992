"""GMAN -- drop-in for torch_geometric_temporal/nn/attention/gman.py: the reference's constructors, attributes, submodule order and
initialisation (xavier_uniform_ conv weights, zero biases), so the state_dict keys
(`_st_att_block1.0._spatial_attention._fully_connected_q._conv2ds.0._conv2d.weight`, ...) and a seeded initialisation equal the
reference's.

Heads: `torch.split(x, K, dim=-1)` cuts the D = K d channels into d heads of width K, head h = channels [h K, (h + 1) K), and the
logits are divided by sqrt(d), the number of heads.  The temporal mask replaces the logits above the diagonal by -32767 after the
scaling; those entries stay inside the softmax sum.  With mask=True and K != d the reference's `mask.repeat(K * batch_size, ...)`
does not broadcast against the d * batch_size attention problems: that RuntimeError is kept, raised before any launch.

The attention core of SpatialAttention, TemporalAttention and TransformAttention (split into heads, Q K^T, the scaling, the mask,
softmax, the product with V and the concatenation of the heads) runs on the fused kernels (DESIGN §4w, stmp_gman_attn_fwd / _bwd), which
read Q, K, V and write O in place in the channels-last (B, T, N, D) activations, when Q, K, V are CUDA float32, K <= 16 and, for the
temporal and transform attentions, both sequence lengths are at most 64; a training call also needs `fused_training`.  Everything else
(float64, longer sequences, wider heads, fused_training = False) runs op for op on the GPU as the reference's algebra:
`spatial_attention_core` and `temporal_attention_core`.

The 1 x 1 convolutions with their BatchNorm stay on PyTorch: each is a row-wise GEMM (F.linear over the contiguous (..., C) rows with
the Conv2d weight viewed as (out, in)) followed by the module's own BatchNorm2d on the rows viewed as a channels-last (1, C, R, 1)
image, which keeps the batch statistics over all R = B T N rows, the running statistics and the momentum (bn_decay=None: a cumulative
average) exactly, with no copy."""
from typing import Callable, Optional, Union

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from ... import ops
from ...plan import _require_cuda

MASKED_LOGIT = -(2 ** 15) + 1           # the reference's temporal-mask value
MAX_WIDTH, MAX_SHORT = 16, 64           # head width of the fused kernels; sequence length of the short (temporal / transform) kernel


def conv_block(X: torch.Tensor, conv: nn.Conv2d, bn: nn.BatchNorm2d, activation) -> torch.Tensor:
    """The reference's Conv2D.forward (1 x 1 conv, BatchNorm2d, activation) on the (..., C_in) rows of X."""
    lead = X.shape[:-1]
    W = conv.weight.view(conv.out_channels, conv.in_channels)
    Y = F.linear(X.reshape(-1, X.shape[-1]), W, conv.bias)
    R, C = Y.shape
    # the (R, C) rows as a channels-last (1, C, R, 1) image: BatchNorm2d reduces each channel over the R rows without a copy, and
    # its output permutes back to (R, C) as a view
    Y = bn(Y.view(1, R, 1, C).permute(0, 3, 1, 2)).permute(0, 2, 3, 1).reshape(*lead, C)
    return Y if activation is None else activation(Y)


def spatial_attention_core(query, key, value, K: int, d: int) -> torch.Tensor:
    """SpatialAttention's attention over the nodes, op for op as the reference computes it: (B, T, N, K d) each -> (B, T, N, K d)."""
    batch_size = query.shape[0]
    query = torch.cat(torch.split(query, K, dim=-1), dim=0)
    key = torch.cat(torch.split(key, K, dim=-1), dim=0)
    value = torch.cat(torch.split(value, K, dim=-1), dim=0)
    attention = torch.matmul(query, key.transpose(2, 3))
    attention /= d ** 0.5
    attention = F.softmax(attention, dim=-1)
    X = torch.matmul(attention, value)
    return torch.cat(torch.split(X, batch_size, dim=0), dim=-1)


def temporal_attention_core(query, key, value, K: int, d: int, mask: bool) -> torch.Tensor:
    """TemporalAttention's (and, without mask, TransformAttention's) attention over the steps, op for op as the reference computes it:
    query (B, Tq, N, K d), key and value (B, Tk, N, K d) -> (B, Tq, N, K d)."""
    batch_size, num_step, num_nodes = query.shape[0], query.shape[1], query.shape[2]
    query = torch.cat(torch.split(query, K, dim=-1), dim=0).permute(0, 2, 1, 3)
    key = torch.cat(torch.split(key, K, dim=-1), dim=0).permute(0, 2, 3, 1)
    value = torch.cat(torch.split(value, K, dim=-1), dim=0).permute(0, 2, 1, 3)
    attention = torch.matmul(query, key)
    attention /= d ** 0.5
    if mask:
        m = torch.tril(torch.ones(num_step, num_step, device=query.device))
        m = torch.unsqueeze(torch.unsqueeze(m, dim=0), dim=0).repeat(K * batch_size, num_nodes, 1, 1).to(torch.bool)
        condition = torch.tensor([MASKED_LOGIT], dtype=torch.float32, device=query.device)
        attention = torch.where(m, attention, condition)
    attention = F.softmax(attention, dim=-1)
    X = torch.matmul(attention, value).permute(0, 2, 1, 3)
    return torch.cat(torch.split(X, batch_size, dim=0), dim=-1)


def check_mask(K: int, d: int, batch_size: int, mask: bool):
    """The reference's torch.where(mask, attention, ...) meets a (K B, ...) mask and (d B, ...) logits.  Unless they agree, or the mask
    has one problem and broadcasts, the reference raises (at the where, or at the next layer when the logits have one problem): raise
    that RuntimeError here, before any launch."""
    kb, db = K * batch_size, d * batch_size
    if mask and kb != db and kb != 1:
        raise RuntimeError(f"The size of tensor a ({kb}) must match the size of tensor b ({db}) at non-singleton dimension 0: GMAN's "
                           f"temporal mask needs K == d (K = {K}, d = {d})")


def fused_route(dtype, is_cuda: bool, batch: int, Lq: int, Lk: int, other: int, K: int, d: int, kind: str, mask: bool,
                needs_grad: bool, fused_training: bool) -> bool:
    """Whether one attention call runs on the fused kernels.  kind "spatial": (B, T = other, N = Lq = Lk); "temporal" / "transform":
    (B, Lq or Lk steps, N = other).  The library decides the grid limits (stmp_gman_attn_supported)."""
    if dtype != torch.float32 or not is_cuda or K > MAX_WIDTH or (needs_grad and not fused_training):
        return False
    spatial = kind == "spatial"
    if not spatial and (Lq > MAX_SHORT or Lk > MAX_SHORT):
        return False
    return ops.gman_attn_supported(batch, other, d, K, Lq, Lk, spatial, mask)


def _attention_scale(d: int) -> float:
    """The reference's `attention /= d ** 0.5` on float32 CUDA tensors multiplies by the float32 reciprocal of float32(sqrt(d))."""
    return float(np.float32(1.0) / np.float32(d ** 0.5))


class _Routed:
    """`fused_training` of a module: True (the default) lets training calls of its attentions run on the fused kernels; setting it
    on GMAN or a block sets it on every attention inside."""

    @property
    def fused_training(self) -> bool:
        return all(m._fused for m in self.modules() if isinstance(m, _Attention))

    @fused_training.setter
    def fused_training(self, value: bool):
        for m in self.modules():
            if isinstance(m, _Attention):
                m._fused = bool(value)


class Conv2D(nn.Module):
    def __init__(self, input_dims: int, output_dims: int, kernel_size: Union[tuple, list], stride: Union[tuple, list] = (1, 1),
                 use_bias: bool = True, activation: Optional[Callable[[torch.FloatTensor], torch.FloatTensor]] = F.relu,
                 bn_decay: Optional[float] = None):
        super().__init__()
        self._activation = activation
        self._conv2d = nn.Conv2d(input_dims, output_dims, kernel_size, stride=stride, padding=0, bias=use_bias)
        self._batch_norm = nn.BatchNorm2d(output_dims, momentum=bn_decay)
        torch.nn.init.xavier_uniform_(self._conv2d.weight)
        if use_bias:
            torch.nn.init.zeros_(self._conv2d.bias)
        if tuple(self._conv2d.kernel_size) != (1, 1) or tuple(self._conv2d.stride) != (1, 1):
            raise ValueError("GMAN's Conv2D blocks are 1 x 1 convolutions with stride 1")

    def forward(self, X: torch.FloatTensor) -> torch.FloatTensor:
        return conv_block(X, self._conv2d, self._batch_norm, self._activation)


class FullyConnected(nn.Module):
    def __init__(self, input_dims: Union[int, list], units: Union[int, list], activations, bn_decay: float, use_bias: bool = True):
        super().__init__()
        if isinstance(units, int):
            units, input_dims, activations = [units], [input_dims], [activations]
        assert type(units) == list
        self._conv2ds = nn.ModuleList([
            Conv2D(input_dims=input_dim, output_dims=num_unit, kernel_size=[1, 1], stride=[1, 1], use_bias=use_bias,
                   activation=activation, bn_decay=bn_decay)
            for input_dim, num_unit, activation in zip(input_dims, units, activations)])

    def forward(self, X: torch.FloatTensor) -> torch.FloatTensor:
        for conv in self._conv2ds:
            X = conv(X)
        return X


class SpatioTemporalEmbedding(nn.Module):
    def __init__(self, D: int, bn_decay: float, steps_per_day: int, use_bias: bool = True):
        super().__init__()
        self._fully_connected_se = FullyConnected(input_dims=[D, D], units=[D, D], activations=[F.relu, None], bn_decay=bn_decay,
                                                  use_bias=use_bias)
        self._fully_connected_te = FullyConnected(input_dims=[steps_per_day + 7, D], units=[D, D], activations=[F.relu, None],
                                                  bn_decay=bn_decay, use_bias=use_bias)

    def forward(self, SE: torch.FloatTensor, TE: torch.FloatTensor, T: int) -> torch.FloatTensor:
        """SE (N, D), TE (B, steps, 2) as (day of week, time of day), truncated to int64 -> (B, steps, N, D).  The one-hot is built
        in the FC's dtype, the reference's default dtype wherever the reference runs."""
        _require_cuda(SE, "SE")
        SE = self._fully_connected_se(SE.unsqueeze(0).unsqueeze(0))
        TE = TE.to(SE.device)
        dt = self._fully_connected_te._conv2ds[0]._conv2d.weight.dtype
        dayofweek = F.one_hot(TE[..., 0].to(torch.int64) % 7, 7).to(dt)
        timeofday = F.one_hot(TE[..., 1].to(torch.int64) % T, T).to(dt)
        TE = torch.cat((dayofweek, timeofday), dim=-1).unsqueeze(dim=2)
        TE = self._fully_connected_te(TE)
        return SE + TE


class _Attention(_Routed, nn.Module):
    """The four FullyConnected layers of one GMAN attention and the routing of its attention core."""
    kind = ""

    def __init__(self, K: int, d: int, bn_decay: float, qkv_in: int):
        super().__init__()
        D = K * d
        self._d = d
        self._K = K
        self._fully_connected_q = FullyConnected(input_dims=qkv_in, units=D, activations=F.relu, bn_decay=bn_decay)
        self._fully_connected_k = FullyConnected(input_dims=qkv_in, units=D, activations=F.relu, bn_decay=bn_decay)
        self._fully_connected_v = FullyConnected(input_dims=qkv_in, units=D, activations=F.relu, bn_decay=bn_decay)
        self._fully_connected = FullyConnected(input_dims=D, units=D, activations=F.relu, bn_decay=bn_decay)
        self._fused = True

    def _core(self, query, key, value, mask: bool = False) -> torch.Tensor:
        spatial = self.kind == "spatial"
        B, Lq, Lk, other = (query.shape[0], query.shape[2], key.shape[2], query.shape[1]) if spatial else \
            (query.shape[0], query.shape[1], key.shape[1], query.shape[2])
        needs_grad = torch.is_grad_enabled() and any(t.requires_grad for t in (query, key, value))
        if fused_route(query.dtype, query.is_cuda, B, Lq, Lk, other, self._K, self._d, self.kind, mask, needs_grad, self._fused) \
                and key.dtype == value.dtype == torch.float32:
            return ops.gman_attention(query, key, value, self._d, self._K, _attention_scale(self._d), spatial, mask, needs_grad)
        if spatial:
            return spatial_attention_core(query, key, value, self._K, self._d)
        return temporal_attention_core(query, key, value, self._K, self._d, mask)


class SpatialAttention(_Attention):
    kind = "spatial"

    def __init__(self, K: int, d: int, bn_decay: float):
        super().__init__(K, d, bn_decay, 2 * K * d)

    def forward(self, X: torch.FloatTensor, STE: torch.FloatTensor) -> torch.FloatTensor:
        _require_cuda(X, "X")
        X = torch.cat((X, STE), dim=-1)
        X = self._core(self._fully_connected_q(X), self._fully_connected_k(X), self._fully_connected_v(X))
        return self._fully_connected(X)


class TemporalAttention(_Attention):
    kind = "temporal"

    def __init__(self, K: int, d: int, bn_decay: float, mask: bool):
        super().__init__(K, d, bn_decay, 2 * K * d)
        self._mask = mask

    def forward(self, X: torch.FloatTensor, STE: torch.FloatTensor) -> torch.FloatTensor:
        _require_cuda(X, "X")
        check_mask(self._K, self._d, X.shape[0], self._mask)
        X = torch.cat((X, STE), dim=-1)
        X = self._core(self._fully_connected_q(X), self._fully_connected_k(X), self._fully_connected_v(X), self._mask)
        return self._fully_connected(X)


class GatedFusion(nn.Module):
    def __init__(self, D: int, bn_decay: float):
        super().__init__()
        self._fully_connected_xs = FullyConnected(input_dims=D, units=D, activations=None, bn_decay=bn_decay, use_bias=False)
        self._fully_connected_xt = FullyConnected(input_dims=D, units=D, activations=None, bn_decay=bn_decay, use_bias=True)
        self._fully_connected_h = FullyConnected(input_dims=[D, D], units=[D, D], activations=[F.relu, None], bn_decay=bn_decay)

    def forward(self, HS: torch.FloatTensor, HT: torch.FloatTensor) -> torch.FloatTensor:
        XS = self._fully_connected_xs(HS)
        XT = self._fully_connected_xt(HT)
        z = torch.sigmoid(torch.add(XS, XT))
        H = torch.add(torch.mul(z, HS), torch.mul(1 - z, HT))
        return self._fully_connected_h(H)


class SpatioTemporalAttention(_Routed, nn.Module):
    def __init__(self, K: int, d: int, bn_decay: float, mask: bool):
        super().__init__()
        self._spatial_attention = SpatialAttention(K, d, bn_decay)
        self._temporal_attention = TemporalAttention(K, d, bn_decay, mask=mask)
        self._gated_fusion = GatedFusion(K * d, bn_decay)

    def forward(self, X: torch.FloatTensor, STE: torch.FloatTensor) -> torch.FloatTensor:
        _require_cuda(X, "X")
        check_mask(self._temporal_attention._K, self._temporal_attention._d, X.shape[0], self._temporal_attention._mask)
        HS = self._spatial_attention(X, STE)
        HT = self._temporal_attention(X, STE)
        H = self._gated_fusion(HS, HT)
        return torch.add(X, H)


class TransformAttention(_Attention):
    kind = "transform"

    def __init__(self, K: int, d: int, bn_decay: float):
        super().__init__(K, d, bn_decay, K * d)

    def forward(self, X: torch.FloatTensor, STE_his: torch.FloatTensor, STE_pred: torch.FloatTensor) -> torch.FloatTensor:
        _require_cuda(X, "X")
        X = self._core(self._fully_connected_q(STE_pred), self._fully_connected_k(STE_his), self._fully_connected_v(X))
        return self._fully_connected(X)


class GMAN(_Routed, nn.Module):
    def __init__(self, L: int, K: int, d: int, num_his: int, bn_decay: float, steps_per_day: int, use_bias: bool, mask: bool):
        super().__init__()
        D = K * d
        self._num_his = num_his
        self._steps_per_day = steps_per_day
        self._st_embedding = SpatioTemporalEmbedding(D, bn_decay, steps_per_day, use_bias)
        self._st_att_block1 = nn.ModuleList([SpatioTemporalAttention(K, d, bn_decay, mask) for _ in range(L)])
        self._st_att_block2 = nn.ModuleList([SpatioTemporalAttention(K, d, bn_decay, mask) for _ in range(L)])
        self._transform_attention = TransformAttention(K, d, bn_decay)
        self._fully_connected_1 = FullyConnected(input_dims=[1, D], units=[D, D], activations=[F.relu, None], bn_decay=bn_decay)
        self._fully_connected_2 = FullyConnected(input_dims=[D, D], units=[D, 1], activations=[F.relu, None], bn_decay=bn_decay)
        self._K, self._d, self._mask = K, d, mask

    def forward(self, X: torch.FloatTensor, SE: torch.FloatTensor, TE: torch.FloatTensor) -> torch.FloatTensor:
        """X (B, num_his, N), SE (N, K d), TE (B, num_his + num_pred, 2) -> (B, num_pred, N)."""
        _require_cuda(X, "X")
        check_mask(self._K, self._d, X.shape[0], self._mask)
        X = self._fully_connected_1(torch.unsqueeze(X, -1))
        STE = self._st_embedding(SE, TE, self._steps_per_day)
        STE_his = STE[:, : self._num_his]
        STE_pred = STE[:, self._num_his:]
        for net in self._st_att_block1:
            X = net(X, STE_his)
        X = self._transform_attention(X, STE_his, STE_pred)
        for net in self._st_att_block2:
            X = net(X, STE_pred)
        return torch.squeeze(self._fully_connected_2(X), 3)
