"""raft_b200 -- H100-native RAO-solve hot path behind the RAFT API (see DESIGN.md).

Importing the package loads ``csrc/libraftk.so`` (sm_90a).  There is no CPU fallback: a missing
library is an ImportError."""
from . import _lib  # noqa: F401  (fails loudly when the CUDA library has not been built)
from . import bem, grid, packer, solver, sweep  # noqa: F401
from .fowt import FOWT  # noqa: F401
from .member import Member  # noqa: F401
from .model import Model  # noqa: F401

__version__ = "0.1.0"
