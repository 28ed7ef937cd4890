"""torchdiffeq_b200 -- an H100-native (sm_90a) implementation of torchdiffeq's explicit Runge-Kutta
hot path behind the reference's own API: odeint / odeint_adjoint(func, y0, t, method=, rtol=, atol=).

Importing the package does not need a GPU; calling a solver does, and fails loudly when libtdq.so is
missing -- there is no CPU or PyTorch fallback."""
from .odeint import odeint, odeint_event, odeint_dense, clear_cache, set_cache_size, last_stats
from .adjoint import odeint_adjoint, find_parameters
from .fields import LinearField
from ._engine import SolverFailure
from ._compact import active_rows
from ._lib import TdqError

__version__ = "0.2.0"
__all__ = ["odeint", "odeint_adjoint", "odeint_event", "odeint_dense", "find_parameters", "clear_cache", "set_cache_size", "last_stats",
           "active_rows", "LinearField", "SolverFailure", "TdqError"]
