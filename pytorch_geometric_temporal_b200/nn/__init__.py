from .recurrent import *  # noqa: F401,F403
from .attention import *  # noqa: F401,F403
from .hetero import *  # noqa: F401,F403
