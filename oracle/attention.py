"""Functional CPU restatement of nn/attention/astgcn.py (oracle; test infrastructure).
``p`` carries the reference module's state_dict keys."""
from typing import Optional

import torch
import torch.nn.functional as F

from . import pyg
from .recurrent import _sub


def cheb_att_norm(edge_index, num_nodes, edge_weight, normalization, lambda_max, dtype=torch.float32, batch=None):
    """ChebConvAttention.__norm__ (astgcn.py:82-110): remove loops -> get_laplacian (appends N loops)
    -> [per-graph lambda_max[batch[row]], :98-99] -> 2w/lam, inf->0 -> add_self_loops(fill=-1) (appends N MORE loops)."""
    ei, ew = pyg.remove_self_loops(edge_index, edge_weight)
    ei, ew = pyg.get_laplacian(ei, ew, normalization, dtype, num_nodes)
    if batch is not None and lambda_max.numel() > 1:
        lambda_max = lambda_max[batch[ei[0]]]
    ew = (2.0 * ew) / lambda_max
    ew = ew.masked_fill(ew == float("inf"), 0)
    return pyg.add_self_loops(ei, ew, fill_value=-1.0, num_nodes=num_nodes)


def cheb_conv_attention(p, x, edge_index, S, normalization=None, edge_weight=None, lambda_max=None, batch=None):
    """ChebConvAttention.forward (astgcn.py:112-183).  x (B,N,Fin), S (B,N,N)."""
    if normalization != "sym" and lambda_max is None:
        raise ValueError("You need to pass `lambda_max` to `forward() in`case the normalization is non-symmetric.")
    if lambda_max is None:
        lambda_max = torch.tensor(2.0, dtype=x.dtype)
    if not isinstance(lambda_max, torch.Tensor):
        lambda_max = torch.tensor(lambda_max, dtype=x.dtype)
    ei, norm = cheb_att_norm(edge_index, x.size(-2), edge_weight, normalization, lambda_max, x.dtype, batch)
    row, col = ei[0], ei[1]
    att = norm * S[:, row, col]                                   # (B,E2)            :156-157
    T0 = torch.diagonal(S, dim1=1, dim2=2).unsqueeze(-1) * x      # (I*S)^T @ x       :160-165
    W = p["_weight"]
    out = torch.matmul(T0, W[0])
    eiT = ei[[1, 0]]                                              # :167
    T1 = T0
    if W.size(0) > 1:
        T1 = pyg.propagate(eiT, T0, att)
        out = out + torch.matmul(T1, W[1])
    for k in range(2, W.size(0)):
        T2 = 2.0 * pyg.propagate(eiT, T1, norm) - T0              # plain norm        :174-178
        out = out + torch.matmul(T2, W[k])
        T0, T1 = T1, T2
    if p.get("_bias") is not None:
        out = out + p["_bias"]
    return out


def spatial_attention(p, X):
    """astgcn.py:230-262.  X (B,N,F,T) -> (B,N,N), softmax over dim=1."""
    LHS = torch.matmul(torch.matmul(X, p["_W1"]), p["_W2"])
    RHS = torch.matmul(p["_W3"], X).transpose(-1, -2)
    S = torch.matmul(p["_Vs"], torch.sigmoid(torch.matmul(LHS, RHS) + p["_bs"]))
    return F.softmax(S, dim=1)


def temporal_attention(p, X):
    """astgcn.py:295-328.  X (B,N,F,T) -> (B,T,T), softmax over dim=1."""
    LHS = torch.matmul(torch.matmul(X.permute(0, 3, 2, 1), p["_U1"]), p["_U2"])
    RHS = torch.matmul(p["_U3"], X)
    E = torch.matmul(p["_Ve"], torch.sigmoid(torch.matmul(LHS, RHS) + p["_be"]))
    return F.softmax(E, dim=1)


def astgcn_block(p, X, edge_index, normalization, time_strides, lambda_max=None):
    """ASTGCNBlock.forward (astgcn.py:408-481).  edge_index: one tensor, or a list of one per timestep (:442-450) with
    `lambda_max` then a list too (or None).  For normalization != 'sym' the reference computes lambda_max with scipy on
    every call (:437-438); pass it in (tests use the same value on both sides)."""
    B, N, Fi, T = X.shape
    E = temporal_attention(_sub(p, "_temporal_attention."), X)
    Xt = torch.matmul(X.reshape(B, -1, T), E).reshape(B, N, Fi, T)
    S = spatial_attention(_sub(p, "_spatial_attention."), Xt)
    lam = lambda ei: pyg.LaplacianLambdaMax()(pyg.Data(edge_index=ei, edge_attr=None, num_nodes=N)).lambda_max
    if not isinstance(edge_index, list):
        eis, lams = [edge_index] * T, [lam(edge_index) if normalization != "sym" and lambda_max is None else lambda_max] * T
    else:
        eis = edge_index
        lams = lambda_max if lambda_max is not None else [lam(ei) if normalization != "sym" else None for ei in eis]
    pc = _sub(p, "_chebconv_attention.")
    Xh = [cheb_conv_attention(pc, X[:, :, :, t], eis[t], S, normalization, None, lams[t]).unsqueeze(-1)
          for t in range(T)]
    Xh = F.relu(torch.cat(Xh, dim=-1))
    Xh = F.conv2d(Xh.permute(0, 2, 1, 3), p["_time_convolution.weight"], p["_time_convolution.bias"],
                  stride=(1, time_strides), padding=(0, 1))
    Xr = F.conv2d(X.permute(0, 2, 1, 3), p["_residual_convolution.weight"], p["_residual_convolution.bias"],
                  stride=(1, time_strides))
    Fo = p["_layer_norm.weight"].numel()
    Y = F.layer_norm(F.relu(Xr + Xh).permute(0, 3, 2, 1), (Fo,), p["_layer_norm.weight"], p["_layer_norm.bias"])
    return Y.permute(0, 2, 3, 1)


def astgcn(p, X, edge_index, nb_block, normalization, time_strides, lambda_max=None):
    """ASTGCN.forward (astgcn.py:587-610).  First block strides time by `time_strides`, the rest by 1 (:549-571)."""
    for i in range(nb_block):
        X = astgcn_block(_sub(p, f"_blocklist.{i}."), X, edge_index, normalization,
                         time_strides if i == 0 else 1, lambda_max)
    X = F.conv2d(X.permute(0, 3, 1, 2), p["_final_conv.weight"], p["_final_conv.bias"])
    return X[:, :, :, -1].permute(0, 2, 1)


# ----------------------------------------------------------------------------------------------
# STConv / MSTGCN (SURVEY 8f rank 1)                 nn/attention/stgcn.py, nn/attention/mstgcn.py
# ----------------------------------------------------------------------------------------------
def temporal_conv(p, X):
    """TemporalConv.forward (stgcn.py:28-47): gated 1xk convolution over time; X (B,T,N,C) -> (B,T-k+1,N,C')."""
    Xp = X.permute(0, 3, 2, 1)
    P = F.conv2d(Xp, p["conv_1.weight"], p["conv_1.bias"])
    Q = torch.sigmoid(F.conv2d(Xp, p["conv_2.weight"], p["conv_2.bias"]))
    H = F.relu(P * Q + F.conv2d(Xp, p["conv_3.weight"], p["conv_3.bias"]))
    return H.permute(0, 3, 2, 1)


def stconv(p, X, edge_index, edge_weight=None, normalization="sym", training=True, eps=1e-5):
    """STConv.forward (stgcn.py:131-160): TemporalConv -> ChebConv on every (b,t) slice -> ReLU -> TemporalConv ->
    BatchNorm2d over the node axis (training mode = batch statistics, the module default)."""
    from . import recurrent as R
    T0 = temporal_conv(_sub(p, "_temporal_conv1."), X)
    pc = _sub(p, "_graph_conv.")
    K = len([k for k in pc if k.startswith("lins.")])
    en = pyg.cheb_norm(edge_index, T0.size(-2), edge_weight, normalization, None, X.dtype)
    T = torch.zeros_like(T0)
    for b in range(T0.size(0)):
        for t in range(T0.size(1)):
            T[b][t] = R.cheb_conv(pc, T0[b][t], en, K)
    T = temporal_conv(_sub(p, "_temporal_conv2."), F.relu(T))
    T = T.permute(0, 2, 1, 3)
    T = F.batch_norm(T, None if training else p["_batch_norm.running_mean"], None if training else p["_batch_norm.running_var"],
                     p["_batch_norm.weight"], p["_batch_norm.bias"], training, 0.1, eps)
    return T.permute(0, 2, 1, 3)


def mstgcn_block(p, X, edge_index, time_strides, lambda_max=None):
    """MSTGCNBlock.forward (mstgcn.py:60-122), static edge_index: the (F,B,N,T) -> (N,F,T*B) RESHAPE (:84-88) is a
    reinterpretation, not a transpose -- it is the spec; ChebConv(normalization=None) with scipy lambda_max."""
    from . import recurrent as R
    B, N, Fi, T = X.shape
    lam = lambda ei: lambda_max if lambda_max is not None else \
        pyg.LaplacianLambdaMax()(pyg.Data(edge_index=ei, edge_attr=None, num_nodes=N)).lambda_max
    pc = _sub(p, "_cheb_conv.")
    K = len([k for k in pc if k.startswith("lins.")])
    Ft = p["_time_conv.weight"].size(0)
    if not isinstance(edge_index, list):
        Xt = X.permute(2, 0, 1, 3).reshape(N, Fi, T * B).permute(2, 0, 1)
        en = pyg.cheb_norm(edge_index, N, None, None, lam(edge_index), X.dtype)
        Xt = F.relu(R.cheb_conv(pc, Xt, en, K))
        Xt = Xt.permute(1, 2, 0).reshape(N, Ft, B, T).permute(2, 0, 1, 3)
    else:                                         # per-timestep graphs (:96-115): a genuine per-slice convolution --
        hats = []                                 # NOT the same function as the tensor path above
        for t in range(T):
            lam_t = lambda_max[t] if isinstance(lambda_max, list) else lam(edge_index[t])
            en = pyg.cheb_norm(edge_index[t], N, None, None, lam_t, X.dtype)
            hats.append(R.cheb_conv(pc, X[:, :, :, t], en, K).unsqueeze(-1))
        Xt = F.relu(torch.cat(hats, dim=-1))
    Xt = F.conv2d(Xt.permute(0, 2, 1, 3), p["_time_conv.weight"], p["_time_conv.bias"], stride=(1, time_strides), padding=(0, 1))
    Xr = F.conv2d(X.permute(0, 2, 1, 3), p["_residual_conv.weight"], p["_residual_conv.bias"], stride=(1, time_strides))
    Y = F.layer_norm(F.relu(Xr + Xt).permute(0, 3, 2, 1), (Ft,), p["_layer_norm.weight"], p["_layer_norm.bias"])
    return Y.permute(0, 2, 3, 1)


def mstgcn(p, X, edge_index, nb_block, time_strides, lambda_max=None):
    """MSTGCN.forward (mstgcn.py:181-200).  With a list of per-timestep graphs, `lambda_max` may be a list too (one per graph)."""
    for i in range(nb_block):
        X = mstgcn_block(_sub(p, f"_blocklist.{i}."), X, edge_index, time_strides if i == 0 else 1, lambda_max)
    X = F.conv2d(X.permute(0, 3, 1, 2), p["_final_conv.weight"], p["_final_conv.bias"])
    return X[:, :, :, -1].permute(0, 2, 1)
