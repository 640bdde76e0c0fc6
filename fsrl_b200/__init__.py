"""fsrl_b200 -- H100-native (sm_90a) hot path for safe RL behind FSRL's API surface.

Only the data-parallel hot path of liuzuxin/FSRL lives here (SURVEY.md section 8): rollout
collection + dual GAE, and the constrained policy updates, as hand-written CUDA behind the
C-ABI in include/fsrl_b200.h.  Importing this package requires the built CUDA library.
"""
from . import _lib  # noqa: F401  (fails loudly when libfsrl_b200.so is missing)

__version__ = "0.1.0"
