"""Heterogeneous temporal models (the reference's nn.hetero)."""
from .heterogclstm import HeteroGCLSTM  # noqa: F401
