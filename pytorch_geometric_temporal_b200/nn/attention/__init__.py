from .astgcn import ASTGCN, ASTGCNBlock, ChebConvAttention, SpatialAttention, TemporalAttention  # noqa: F401
from .stgcn import STConv, TemporalConv  # noqa: F401
from .mstgcn import MSTGCN, MSTGCNBlock  # noqa: F401
from .gman import GMAN, SpatioTemporalAttention, SpatioTemporalEmbedding  # noqa: F401
from .mtgnn import MTGNN, GraphConstructor, MixProp  # noqa: F401
