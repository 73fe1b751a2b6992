"""AVWGCN and AGCRN -- drop-ins for torch_geometric_temporal/nn/recurrent/agcrn.py: the reference's constructors and attributes, the
keys `weights_pool (d, K, in, out)` (glorot) and `bias_pool (d, out)` (zeros) under `_gate` and `_update`, created in the reference's
order, so the state_dict keys and a seeded initialisation equal the reference's.

The graph is learned: S = softmax(relu(E E^T), dim=1) over the node embeddings E (N, d), recomputed on every call, with the Chebyshev
supports [I, S, 2 S S - I][:max(K, 2)], and every node has its own weights W_n = E[n] weights_pool and bias E[n] bias_pool.  At K = 1
the support stack still holds [I, S] and the single weight block multiplies Y + S Y, as the reference's einsum broadcast does.  In the
cell Z gates the state inside the candidate and R is the update gate: H' = R H + (1 - R) tanh(AVWGCN_update([X | Z H])).

AGCRN calls run on the fused kernels (DESIGN §4u: stmp_agcrn_fwd, six launches, seven at K = 3; training calls add the hand-written
backward stmp_agcrn_bwd) when X (B, N, in_channels), E (N, d), H and the parameters are float32 and the library supports the shape
(N <= 4096, out_channels <= 64, in_channels + out_channels <= 128, K <= 3, d <= 64, B <= 8 388 607); training calls also need `fused_training`.
Everything else, and AVWGCN called on its own, runs op for op on the GPU: `agcrn_cell` and `avwgcn`, the reference's algebra.

Every call inside the envelope runs fused, which is deliberate: one code path whose every sum has an order fixed by the library, not by
cuBLAS's per-shape algorithm choice, and a training forward equal to the no_grad call bit for bit.  The fused route is about 3x faster
where launches dominate (the tutorial).  On one H100 it is 3-25 % slower than op for op at the paper's shape (B = 64, N = 307, 64
channels) and on 4 096 nodes (DESIGN §4u).  Set `fused_training = False` to send training calls op for op."""
import torch

from ... import ops
from ...plan import _require_cuda
from ._cheb import glorot_


def avwgcn(X: torch.Tensor, E: torch.Tensor, weights_pool: torch.Tensor, bias_pool: torch.Tensor, K: int) -> torch.Tensor:
    """One AVWGCN, op for op on X's device, as the reference computes it: X (B, N, Ci), E (N, d) -> (B, N, Co)."""
    number_of_nodes = E.shape[0]
    supports = torch.softmax(torch.relu(torch.mm(E, E.transpose(0, 1))), dim=1)
    support_set = [torch.eye(number_of_nodes, device=supports.device, dtype=supports.dtype), supports]
    for _ in range(2, K):
        support_set.append(torch.matmul(2 * supports, support_set[-1]) - support_set[-2])
    supports = torch.stack(support_set, dim=0)
    W = torch.einsum("nd,dkio->nkio", E, weights_pool)
    bias = torch.matmul(E, bias_pool)
    X_G = torch.einsum("knm,bmc->bknc", supports, X)
    X_G = X_G.permute(0, 2, 1, 3)
    return torch.einsum("bnki,nkio->bno", X_G, W) + bias


def agcrn_cell(X, E, H, gate, update, out_channels: int) -> torch.Tensor:
    """One AGCRN call op for op on X's device, as the reference computes it: gate / update are the (weights_pool, bias_pool, K) of the
    two AVWGCNs, H (B, N, out) or None (float32 zeros, as the reference's default)."""
    if H is None:
        H = torch.zeros(X.shape[0], X.shape[1], out_channels).to(X.device)
    X_H = torch.cat((X, H), dim=-1)
    Z_R = torch.sigmoid(avwgcn(X_H, E, *gate))
    Z, R = torch.split(Z_R, out_channels, dim=-1)
    C = torch.cat((X, Z * H), dim=-1)
    HC = torch.tanh(avwgcn(C, E, *update))
    return R * H + (1 - R) * HC


class AVWGCN(torch.nn.Module):
    def __init__(self, in_channels: int, out_channels: int, K: int, embedding_dimensions: int):
        super().__init__()
        self.K = K
        self.weights_pool = torch.nn.Parameter(torch.Tensor(embedding_dimensions, K, in_channels, out_channels))
        self.bias_pool = torch.nn.Parameter(torch.Tensor(embedding_dimensions, out_channels))
        glorot_(self.weights_pool)
        with torch.no_grad():
            self.bias_pool.fill_(0)

    def forward(self, X: torch.FloatTensor, E: torch.FloatTensor) -> torch.FloatTensor:
        _require_cuda(X, "X")
        return avwgcn(X, E, self.weights_pool, self.bias_pool, self.K)


class AGCRN(torch.nn.Module):
    def __init__(self, number_of_nodes: int, in_channels: int, out_channels: int, K: int, embedding_dimensions: int):
        super().__init__()
        self.number_of_nodes = number_of_nodes
        self.in_channels = in_channels
        self.out_channels = out_channels
        self.K = K
        self.embedding_dimensions = embedding_dimensions
        self._setup_layers()
        self.fused_training = True      # False: op-for-op autograd path for training calls (tests compare the two)

    def _setup_layers(self):
        self._gate = AVWGCN(in_channels=self.in_channels + self.out_channels, out_channels=2 * self.out_channels, K=self.K,
                            embedding_dimensions=self.embedding_dimensions)
        self._update = AVWGCN(in_channels=self.in_channels + self.out_channels, out_channels=self.out_channels, K=self.K,
                              embedding_dimensions=self.embedding_dimensions)

    def _check(self, X, E, H):
        """The reference's shape errors (its einsum over the nodes, its torch.cat with H), raised before any launch."""
        if X.dim() != 3 or E.dim() != 2 or E.shape[0] != X.shape[1]:
            raise RuntimeError(f"AGCRN: X {tuple(X.shape)} must be (B, N, in_channels) and E {tuple(E.shape)} (N, embedding_dimensions)")
        if H is not None and tuple(H.shape) != (X.shape[0], X.shape[1], self.out_channels):
            raise RuntimeError(f"AGCRN: H {tuple(H.shape)} must be {(X.shape[0], X.shape[1], self.out_channels)}")

    def _fused_ok(self, X, E, H, needs_grad):
        """The module's conditions for the fused kernels (the library decides the widths: stmp_agcrn_supported)."""
        if (needs_grad and not self.fused_training) or X.size(2) != self.in_channels or E.size(1) != self.embedding_dimensions:
            return False
        if any(t.dtype != torch.float32 for t in (X, E, *self.parameters())) or (H is not None and H.dtype != torch.float32):
            return False
        return ops.agcrn_supported(X.shape[0], X.shape[1], self.in_channels, self.out_channels, self.K, self.embedding_dimensions)

    def forward(self, X: torch.FloatTensor, E: torch.FloatTensor, H: torch.FloatTensor = None) -> torch.FloatTensor:
        self._check(X, E, H)
        _require_cuda(X, "X")
        params = (self._gate.weights_pool, self._gate.bias_pool, self._update.weights_pool, self._update.bias_pool)
        needs_grad = torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in (X, E, H, *params))
        if self._fused_ok(X, E, H, needs_grad):
            return ops.agcrn_train(X, E, H, *params) if needs_grad else ops.agcrn_fwd(X, E, H, *params)
        return agcrn_cell(X, E, H, (*params[:2], self.K), (*params[2:], self.K), self.out_channels)
