"""pytorch_geometric_temporal_b200 -- sm_90a (H100) engine behind torch_geometric_temporal's
nn.recurrent / nn.attention forward(X, edge_index, edge_weight, H) surface.  See DESIGN.md."""
__version__ = "0.1.0"

from . import _lib, plan, ops  # noqa: F401
from . import nn, signal  # noqa: F401
