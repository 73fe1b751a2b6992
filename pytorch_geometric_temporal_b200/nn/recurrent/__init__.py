from .dcrnn import DConv, DCRNN, BatchedDConv, BatchedDCRNN  # noqa: F401
from .gconv_gru import GConvGRU  # noqa: F401
from .gconv_lstm import GConvLSTM  # noqa: F401
from .temporalgcn import TGCN, TGCN2  # noqa: F401
from .attentiontemporalgcn import A3TGCN, A3TGCN2  # noqa: F401
from .gc_lstm import GCLSTM  # noqa: F401
from .lrgcn import LRGCN  # noqa: F401
from .dygrae import DyGrEncoder  # noqa: F401
from .evolvegcn import EvolveGCNH, EvolveGCNO  # noqa: F401
from .mpnn_lstm import MPNNLSTM  # noqa: F401
from .agcrn import AGCRN, AVWGCN  # noqa: F401
from ._cheb import ChebConv  # noqa: F401
