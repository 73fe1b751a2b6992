"""ASTGCN -- drop-in for torch_geometric_temporal/nn/attention/astgcn.py (ChebConvAttention :16-199,
SpatialAttention :201-262, TemporalAttention :264-328, ASTGCNBlock :330-481, ASTGCN :483-610).
Same constructors, forward signatures, `__repr__` and state_dict keys (`_blocklist.{i}.
_temporal_attention.{_U1,_U2,_U3,_be,_Ve}`, `._spatial_attention.{_W1,_W2,_W3,_bs,_Vs}`,
`._chebconv_attention.{_weight,_bias}`, `._time_convolution.*`, `._residual_convolution.*`,
`._layer_norm.*`, `_final_conv.*`).

What runs where
* graph work (the hot path): attention-weighted gather/scatter `norm * S[b,row,col]` and the Chebyshev
  recurrence go through `stmp_spmm` on a cached CHEB_ATT plan; the reference's per-timestep Python loop
  (:442-450) is folded into the feature axis (the attention matrix is shared by all T timesteps), so one
  launch per hop covers every timestep; the dense `(I*S)^T @ x` used for a diagonal scale (:160-165) is
  a broadcast multiply;
* inference on a static graph (N <= 1024, T <= 12, 64 time filters, stride 1) keeps the activations channels-last
  (B, N, T, F) between blocks and runs every large product on wgmma with its neighbours fused (csrc/gemm_blocks.cu):
  spatial attention `softmax(Vs @ sigmoid(LHS @ RHS + bs))` in ONE kernel up to 320 nodes (the N x N sigmoid is generated in
  the operand stage, the softmax is the epilogue; the result is kept transposed and consumed so by `stmp_spmm_att_t`), and
  above that in a column-tiled pair whose second launch normalises the rows (csrc/spatial_attention_tiled.cu); the Chebyshev
  contraction + ReLU; time convolution + residual convolution + ReLU + LayerNorm; the final convolution; and the small-matrix
  front (temporal attention, X~ = X E, the (B,N,T) attention factors) in one launch (`stmp_astgcn_factors_fwd`).  No
  im2col, cat or permute of activations in HBM;
* training (autograd) and the per-timestep edge_index list path use the op-for-op torch formulation around `stmp_spmm`
  (dense products on cuBLAS through torch).
* lambda_max for normalization != "sym": the reference calls scipy ARPACK on the host in EVERY block
  forward (:437-438); here it is computed once per static graph and cached.
"""
from typing import List, Optional, Union

import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.nn import Parameter

from ... import _lib, ops
from ...plan import PlanCache, _require_cuda


def laplacian_lambda_max(edge_index: torch.Tensor, num_nodes: int, normalization: Optional[str]) -> float:
    """torch_geometric.transforms.LaplacianLambdaMax (is_undirected=False): largest-magnitude eigenvalue of
    the (normalised) Laplacian via scipy `eigs`.  One-time host computation per static graph."""
    import numpy as np
    from scipy.sparse import coo_matrix
    from scipy.sparse.linalg import eigs
    ei = edge_index.detach().cpu()
    keep = ei[0] != ei[1]
    row, col = ei[0][keep].numpy(), ei[1][keep].numpy()
    w = np.ones(row.shape[0], dtype=np.float64)
    deg = np.bincount(row, weights=w, minlength=num_nodes)
    if normalization is None:
        vals, r, c = np.concatenate([-w, deg]), np.concatenate([row, np.arange(num_nodes)]), np.concatenate([col, np.arange(num_nodes)])
    else:
        with np.errstate(divide="ignore"):
            if normalization == "sym":
                d = np.where(deg > 0, deg ** -0.5, 0.0)
                wn = d[row] * w * d[col]
            else:
                d = np.where(deg > 0, 1.0 / deg, 0.0)
                wn = d[row] * w
        vals = np.concatenate([-wn, np.ones(num_nodes)])
        r, c = np.concatenate([row, np.arange(num_nodes)]), np.concatenate([col, np.arange(num_nodes)])
    L = coo_matrix((vals.astype(np.float32).astype(np.float64), (r, c)), shape=(num_nodes, num_nodes))
    lam = eigs(L, k=1, which="LM", return_eigenvectors=False)
    return float(lam.real[0])


class ChebConvAttention(nn.Module):
    def __init__(self, in_channels: int, out_channels: int, K: int, normalization: Optional[str] = None, bias: bool = True,
                 **kwargs):
        super().__init__()
        assert K > 0
        assert normalization in [None, "sym", "rw"], "Invalid normalization"
        self._in_channels, self._out_channels, self._normalization = in_channels, out_channels, normalization
        self._weight = Parameter(torch.empty(K, in_channels, out_channels))
        if bias:
            self._bias = Parameter(torch.empty(out_channels))
        else:
            self.register_parameter("_bias", None)
        self._plans = PlanCache(max_entries=16)
        self._reset_parameters()

    def _reset_parameters(self):
        nn.init.xavier_uniform_(self._weight)
        if self._bias is not None:
            nn.init.uniform_(self._bias)

    def _plan(self, edge_index, edge_weight, num_nodes, lambda_max, batch=None):
        if batch is not None and torch.is_tensor(lambda_max) and lambda_max.numel() > 1:     # astgcn.py:98-99
            return self._plans.get(_lib.FLAVOR_CHEB_ATT, edge_index, edge_weight, num_nodes, self._normalization, lambda_max, batch=batch)
        lam = None if lambda_max is None else float(lambda_max)
        return self._plans.get(_lib.FLAVOR_CHEB_ATT, edge_index, edge_weight, num_nodes, self._normalization, lam)

    def forward(self, x: torch.FloatTensor, edge_index: torch.LongTensor, spatial_attention: torch.FloatTensor,
                edge_weight=None, batch=None, lambda_max=None) -> torch.FloatTensor:
        """x (B,N,Fin) -- or (B,N,T,Fin) to process every timestep of a block in one pass --,
        spatial_attention (B,N,N) -> (B,N,[T,]Fout)."""
        if self._normalization != "sym" and lambda_max is None:
            raise ValueError("You need to pass `lambda_max` to `forward() in`case the normalization is non-symmetric.")
        _require_cuda(x, "x")
        B, N = x.shape[0], x.shape[1]
        # `batch` (node -> graph id of a multi-graph mini-batch) only selects the per-graph lambda_max (astgcn.py:98-99)
        plan = self._plan(edge_index, edge_weight, N, lambda_max, batch)
        xs = x.reshape(B, N, -1)                                    # timesteps folded into the feature axis
        S = spatial_attention.contiguous()
        T0 = torch.diagonal(S, dim1=1, dim2=2).unsqueeze(-1) * xs   # (I*S)^T @ x            :160-165
        Ts = [T0]
        K = self._weight.size(0)
        if K > 1:
            Ts.append(ops.spmm(plan, 0, T0.contiguous(), att=S))   # norm * S[b,row,col]    :156-157,169-171
        for _ in range(2, K):
            Ts.append(ops.spmm(plan, 0, Ts[-1], alpha=2.0, z=Ts[-2], beta=-1.0))   # plain norm   :174-178
        out = 0
        for k in range(K):
            out = out + torch.matmul(Ts[k].reshape(x.shape), self._weight[k])
        if self._bias is not None:
            out = out + self._bias
        return out

    def __repr__(self):
        return "{}({}, {}, K={}, normalization={})".format(self.__class__.__name__, self._in_channels, self._out_channels,
                                                           self._weight.size(0), self._normalization)


class SpatialAttention(nn.Module):
    def __init__(self, in_channels: int, num_of_vertices: int, num_of_timesteps: int):
        super().__init__()
        self._W1 = nn.Parameter(torch.FloatTensor(num_of_timesteps))
        self._W2 = nn.Parameter(torch.FloatTensor(in_channels, num_of_timesteps))
        self._W3 = nn.Parameter(torch.FloatTensor(in_channels))
        self._bs = nn.Parameter(torch.FloatTensor(1, num_of_vertices, num_of_vertices))
        self._Vs = nn.Parameter(torch.FloatTensor(num_of_vertices, num_of_vertices))
        _reset(self)

    def forward(self, X: torch.FloatTensor) -> torch.FloatTensor:
        LHS = torch.matmul(torch.matmul(X, self._W1), self._W2)
        RHS = torch.matmul(self._W3, X).transpose(-1, -2)
        S = torch.matmul(self._Vs, torch.sigmoid(torch.matmul(LHS, RHS) + self._bs))
        return F.softmax(S, dim=1)


class TemporalAttention(nn.Module):
    def __init__(self, in_channels: int, num_of_vertices: int, num_of_timesteps: int):
        super().__init__()
        self._U1 = nn.Parameter(torch.FloatTensor(num_of_vertices))
        self._U2 = nn.Parameter(torch.FloatTensor(in_channels, num_of_vertices))
        self._U3 = nn.Parameter(torch.FloatTensor(in_channels))
        self._be = nn.Parameter(torch.FloatTensor(1, num_of_timesteps, num_of_timesteps))
        self._Ve = nn.Parameter(torch.FloatTensor(num_of_timesteps, num_of_timesteps))
        _reset(self)

    def forward(self, X: torch.FloatTensor) -> torch.FloatTensor:
        LHS = torch.matmul(torch.matmul(X.permute(0, 3, 2, 1), self._U1), self._U2)
        RHS = torch.matmul(self._U3, X)
        E = torch.matmul(self._Ve, torch.sigmoid(torch.matmul(LHS, RHS) + self._be))
        return F.softmax(E, dim=1)


def _conv_1xk(conv: nn.Conv2d, x: torch.Tensor) -> torch.Tensor:
    """Conv2d with a (1,k) kernel, stride (1,s), padding (0,p) on (B,C,N,T) as an fp32 contraction.
    cuDNN convolutions default to TF32 (torch.backends.cudnn.allow_tf32=True) in forward AND backward, which
    misses the strict fp32 parity tolerance; unfold + einsum runs on fp32 cuBLAS and keeps the Conv2d
    parameters (state_dict layout unchanged)."""
    k, s_, p_ = conv.kernel_size[1], conv.stride[1], conv.padding[1]
    if p_:
        x = F.pad(x, (p_, p_))
    w = conv.weight[:, :, 0, :]                                  # (O, C, k)
    if k == 1:
        out = torch.einsum("bcnt,oc->bont", x[..., ::s_], w[:, :, 0])
    else:
        out = torch.einsum("bcntk,ock->bont", x.unfold(-1, k, s_), w)
    if conv.bias is not None:
        out = out + conv.bias.view(1, -1, 1, 1)
    return out


def _needs_grad(module, *tensors):
    if not torch.is_grad_enabled():
        return False
    return any(p.requires_grad for p in module.parameters()) or any(t.requires_grad for t in tensors)


def _reset(module):
    """xavier_uniform for dim>1, uniform(0,1) otherwise -- applied to EVERY parameter (astgcn.py:401-406)."""
    for p in module.parameters():
        if p.dim() > 1:
            nn.init.xavier_uniform_(p)
        else:
            nn.init.uniform_(p)


class ASTGCNBlock(nn.Module):
    def __init__(self, in_channels: int, K: int, nb_chev_filter: int, nb_time_filter: int, time_strides: int,
                 num_of_vertices: int, num_of_timesteps: int, normalization: Optional[str] = None, bias: bool = True):
        super().__init__()
        self._temporal_attention = TemporalAttention(in_channels, num_of_vertices, num_of_timesteps)
        self._spatial_attention = SpatialAttention(in_channels, num_of_vertices, num_of_timesteps)
        self._chebconv_attention = ChebConvAttention(in_channels, nb_chev_filter, K, normalization, bias)
        self._time_convolution = nn.Conv2d(nb_chev_filter, nb_time_filter, kernel_size=(1, 3), stride=(1, time_strides), padding=(0, 1))
        self._residual_convolution = nn.Conv2d(in_channels, nb_time_filter, kernel_size=(1, 1), stride=(1, time_strides))
        self._layer_norm = nn.LayerNorm(nb_time_filter)
        self._normalization = normalization
        self._lam_cache = {}
        _reset(self)

    def _lambda_max(self, edge_index, num_nodes):
        if self._normalization == "sym":
            return None
        key = (edge_index.data_ptr(), edge_index._version, tuple(edge_index.shape))
        hit = self._lam_cache.get(key)
        if hit is None:
            if len(self._lam_cache) > 16:
                self._lam_cache.clear()
            # the reference calls LaplacianLambdaMax() with ITS default normalization=None whatever the block's
            # normalization is (astgcn.py:437-438): lambda_max of L = D - A.  Reproduced.
            hit = (laplacian_lambda_max(edge_index, num_nodes, None), edge_index)
            self._lam_cache[key] = hit
        return hit[0]

    # ---- native inference path: channels-last activations, fused wgmma products ------------------------------------
    def _native_ok(self, N, Fi, T):
        tc, rc = self._time_convolution, self._residual_convolution
        ta, sa = self._temporal_attention, self._spatial_attention
        K = self._chebconv_attention._weight.size(0)
        # the kernels take N, Fi and T from X and index the parameters with them: an X of another shape goes to the op-for-op path,
        # which raises the reference's shape error
        shapes_match = (ta._U1.shape == (N,) and ta._U3.shape == (Fi,) and ta._be.shape == (1, T, T) and sa._Vs.shape == (N, N))
        return (shapes_match and N <= 1024 and T <= 12 and Fi <= 64 and K <= 12 and tc.out_channels == 64 and tc.in_channels == 64
                and tc.stride[1] == 1 and rc.stride[1] == 1 and tc.kernel_size == (1, 3) and tc.padding == (0, 1))

    def _native_packs(self):
        def build():
            ta, sa, cc = self._temporal_attention, self._spatial_attention, self._chebconv_attention
            tc, rc = self._time_convolution, self._residual_convolution
            K = cc._weight.size(0)
            return dict(
                vsT=ops.spatial_attention_prepack(sa._Vs), bsT=sa._bs[0].t().contiguous(),
                cheb=ops.gemm_blocks_prepack([cc._weight[k] for k in range(K)]),                       # (Fi, Fc) per hop
                # time conv taps t-1, t, t+1: W[o, c, 0, tap] -> (c, o); residual 1x1: W[o, c, 0, 0] -> (c, o)
                tconv=ops.gemm_blocks_prepack([tc.weight[:, :, 0, j].t().contiguous() for j in range(3)]
                                              + [rc.weight[:, :, 0, 0].t().contiguous()]),
                tbias=(tc.bias + rc.bias).contiguous())
        if not hasattr(self, "_npack"):
            self._npack = ops.PackCache()
        return self._npack.get(list(self.parameters()), build)

    def forward_channels_last(self, Xc: torch.Tensor, edge_index: torch.Tensor) -> torch.Tensor:
        """Xc (B, N, T, Fi) contiguous -> (B, N, T, Ft) contiguous; inference only (no autograd)."""
        B, N, T, Fi = Xc.shape
        ta, sa, cc = self._temporal_attention, self._spatial_attention, self._chebconv_attention
        pk = self._native_packs()
        # temporal attention (astgcn.py:311-328), X~ = X E (:427-430) and the spatial-attention factors (:245-256): one launch
        try:
            lhs_s, rhs_s = ops.astgcn_factors(Xc, ta._U1, ta._U2, ta._U3, ta._be, ta._Ve, sa._W1, sa._W2, sa._W3)
        except _lib.StmpUnsupported:         # odd channel counts: the same algebra on torch
            lhs = torch.matmul(torch.einsum("bntf,n->btf", Xc, ta._U1), ta._U2)                # (B,T,N)
            rhs = torch.einsum("bntf,f->bnt", Xc, ta._U3)                                       # (B,N,T)
            E = F.softmax(torch.matmul(ta._Ve, torch.sigmoid(torch.matmul(lhs, rhs) + ta._be)), dim=1)
            Xt = torch.einsum("bntf,btu->bnuf", Xc, E)                                          # X~ channels-last
            lhs_s = torch.matmul(torch.einsum("bnuf,u->bnf", Xt, sa._W1), sa._W2)               # (B,N,T)
            rhs_s = torch.einsum("bnuf,f->bun", Xt, sa._W3).contiguous()                        # (B,T,N)
        # the fused N x N kernel; ST[b, j, i] = S[b, i, j]
        ST = ops.spatial_attention(lhs_s, rhs_s, pk["bsT"], pk["vsT"])
        # ChebConvAttention over all T timesteps at once (:141-183): T_0 = diag(S) x, T_1 = (norm * S) T_0, T_k = 2 L T_{k-1} - T_{k-2}
        lam = self._lambda_max(edge_index, N)
        if cc._normalization != "sym" and lam is None:
            raise ValueError("You need to pass `lambda_max` to `forward() in`case the normalization is non-symmetric.")
        plan = cc._plan(edge_index, None, N, lam)
        K = cc._weight.size(0)
        x2 = Xc.reshape(B, N, T * Fi)
        Ts = [torch.diagonal(ST, dim1=1, dim2=2)[:, :N].unsqueeze(-1) * x2]
        if K > 1:
            Ts.append(ops.spmm_attT(plan, 0, Ts[0], ST))
        for _ in range(2, K):
            Ts.append(ops.spmm_raw(plan, 0, Ts[-1], alpha=2.0, z=Ts[-2], beta=-1.0))
        Fc = cc._weight.size(2)
        Xh = ops.gemm_blocks([(t.reshape(B * N * T, Fi), Fi, 0) for t in Ts], pk["cheb"], 64, Fc, cc._bias, ops.EPI_RELU)   # (BNT, Fc)
        # time conv (1x3, pad 1) + residual 1x1 conv + ReLU + LayerNorm (:473-480) in one launch
        Xf = Xc.reshape(B * N * T, Fi)
        ln = self._layer_norm
        Y = ops.gemm_blocks([(Xh, Fc, -1), (Xh, Fc, 0), (Xh, Fc, 1), (Xf, Fi, 0)], pk["tconv"], 64, 64, pk["tbias"], ops.EPI_RELU_LN,
                            ln.weight, ln.bias, ln.eps, seq=T)
        return Y.view(B, N, T, 64)

    def forward(self, X: torch.FloatTensor, edge_index: Union[torch.LongTensor, List[torch.LongTensor]]) -> torch.FloatTensor:
        B, N, Fi, T = X.shape
        if (not isinstance(edge_index, list)) and self._native_ok(N, Fi, T) and not _needs_grad(self, X):
            return self.forward_channels_last(X.permute(0, 1, 3, 2).contiguous(), edge_index).permute(0, 1, 3, 2)
        E = self._temporal_attention(X)
        X_tilde = torch.matmul(X.reshape(B, -1, T), E).reshape(B, N, Fi, T)
        S = self._spatial_attention(X_tilde)
        if not isinstance(edge_index, list):
            lam = self._lambda_max(edge_index, N)
            # all T timesteps in one pass: (B,N,F,T) -> (B,N,T,F)
            X_hat = self._chebconv_attention(X.permute(0, 1, 3, 2).contiguous(), edge_index, S, lambda_max=lam)
            X_hat = F.relu(X_hat.permute(0, 1, 3, 2))             # (B,N,Fc,T)
        else:
            hats = []
            for t in range(T):
                lam = self._lambda_max(edge_index[t], N)
                hats.append(self._chebconv_attention(X[:, :, :, t].contiguous(), edge_index[t], S, lambda_max=lam).unsqueeze(-1))
            X_hat = F.relu(torch.cat(hats, dim=-1))
        X_hat = _conv_1xk(self._time_convolution, X_hat.permute(0, 2, 1, 3))
        Xr = _conv_1xk(self._residual_convolution, X.permute(0, 2, 1, 3))
        Y = self._layer_norm(F.relu(Xr + X_hat).permute(0, 3, 2, 1))
        return Y.permute(0, 2, 3, 1)


class ASTGCN(nn.Module):
    def __init__(self, nb_block: int, in_channels: int, K: int, nb_chev_filter: int, nb_time_filter: int, time_strides: int,
                 num_for_predict: int, len_input: int, num_of_vertices: int, normalization: Optional[str] = None,
                 bias: bool = True):
        super().__init__()
        self._blocklist = nn.ModuleList([ASTGCNBlock(in_channels, K, nb_chev_filter, nb_time_filter, time_strides,
                                                     num_of_vertices, len_input, normalization, bias)])
        self._blocklist.extend([ASTGCNBlock(nb_time_filter, K, nb_chev_filter, nb_time_filter, 1, num_of_vertices,
                                            len_input // time_strides, normalization, bias) for _ in range(nb_block - 1)])
        self._final_conv = nn.Conv2d(int(len_input / time_strides), num_for_predict, kernel_size=(1, nb_time_filter))
        _reset(self)

    def _final_pack(self):
        def build():
            w = self._final_conv.weight                                      # (P, T', 1, Ft)
            blocks = [w[:, t, 0, :].t().contiguous() for t in range(w.size(1))]   # per timestep (Ft, P)
            P = w.size(0)
            P16 = (P + 15) // 16 * 16
            blocks = [F.pad(b, (0, P16 - P)) for b in blocks]
            bias = F.pad(self._final_conv.bias, (0, P16 - P))
            return ops.gemm_blocks_prepack(blocks), bias.contiguous(), P16
        if not hasattr(self, "_fpack"):
            self._fpack = ops.PackCache()
        return self._fpack.get(list(self._final_conv.parameters()), build)

    def forward(self, X: torch.FloatTensor, edge_index: torch.LongTensor) -> torch.FloatTensor:
        _require_cuda(X, "X")
        B, N, Fi, T = X.shape
        fc = self._final_conv
        # the final convolution is one blocked GEMM of num_for_predict (rounded up to 16) <= 320 output columns
        if (not isinstance(edge_index, list) and not _needs_grad(self, X) and fc.in_channels <= 12 and fc.kernel_size[1] == 64
                and fc.out_channels <= 320 and all(b._native_ok(N, Fi if i == 0 else 64, T) for i, b in enumerate(self._blocklist))):
            # inference: channels-last (B,N,T,F) all the way, one layout change at the input
            Xc = X.permute(0, 1, 3, 2).contiguous()
            for block in self._blocklist:
                Xc = block.forward_channels_last(Xc, edge_index)
            packed, bias, P16 = self._final_pack()
            Tn = Xc.size(2)
            rows = Xc.reshape(B * N, Tn * 64)
            out = ops.gemm_blocks([(rows[:, 64 * t:64 * t + 64], 64, 0) for t in range(Tn)], packed, P16, fc.out_channels, bias, ops.EPI_BIAS)
            return out.view(B, N, fc.out_channels)
        for block in self._blocklist:
            X = block(X, edge_index)
        X = _conv_1xk(self._final_conv, X.permute(0, 3, 1, 2))     # kernel (1, F_t) over the feature axis
        return X[:, :, :, -1].permute(0, 2, 1)
