"""Drop-ins for the ``ding.torch_utils`` modules behind the reference's plugin registry (ding/hpc_rl/wrapper.py:62-73)."""
from .lstm import LSTM
from .scatter_connection import ScatterConnection

__all__ = ['LSTM', 'ScatterConnection']
