"""The layer-normalised LSTM of ding/torch_utils/network/rnn.py:131-239 (``lstm_type='normal'``, ``norm_type='LN'``), the
recurrent core of DRQN, R2D2, R2D3 and NGU.  Each layer of each call is one ``ops.LNLSTMFunction``: the GEMMs go to cuBLAS
through torch.mm, everything between them runs on csrc/lstm.cu, one launch per step in each direction.

``LSTM`` is a standalone drop-in with the reference's constructor, parameter names and initialisation order, so that a
``state_dict`` loads both ways and one seed draws the same weights.  ``patched_forward`` is what ``install()`` sets as
``forward`` on the reference class: it keeps the instance's own state handling and hands the call to the original forward
when the inputs, weights or norms are not the ones the kernels compute (CUDA fp32, ``nn.LayerNorm`` with eps 1e-5 and an
affine transform).
"""
import math
from typing import Dict, List, Optional, Tuple, Union

import torch
import torch.nn as nn

from .. import ops, torch_ops

LN_EPS = 1e-5  # the eps csrc/lstm.cu normalises with: nn.LayerNorm's default


def _fp32_on(t, device):
    return isinstance(t, torch.Tensor) and t.dtype == torch.float32 and t.device == device


def accelerated(m, inputs) -> bool:
    """whether the kernels compute ``m``'s forward on ``inputs``: CUDA fp32 input and weights, affine LayerNorms"""
    if not (isinstance(inputs, torch.Tensor) and inputs.is_cuda and inputs.dtype == torch.float32 and inputs.dim() == 3):
        return False
    dev, G = inputs.device, 4 * m.hidden_size
    if not (_fp32_on(m.bias, dev) and all(_fp32_on(w, dev) for w in list(m.wx) + list(m.wh))):
        return False
    for n in m.norm:
        if type(n) is not nn.LayerNorm or n.eps != LN_EPS or tuple(n.normalized_shape) != (G, ):
            return False
        if not (_fp32_on(n.weight, dev) and _fp32_on(n.bias, dev)):
            return False
    return True


def _state_ok(m, state, inputs) -> bool:
    shape = (m.num_layers, inputs.shape[1], m.hidden_size)
    return len(state) == 2 and all(_fp32_on(s, inputs.device) and tuple(s.shape) == shape for s in state)


def layers(m, inputs, H0, C0):
    """the layer loop of rnn.py:212-236 on the kernels -> (output (T, B, H), [h (L, B, H), c (L, B, H)]); dropout between
    layers goes through ``m.dropout`` where the reference applies it, so one seed gives the same masks"""
    x = inputs
    hs, cs = [], []
    grad = torch.is_grad_enabled()
    for l in range(m.num_layers):
        nx, nh = m.norm[2 * l], m.norm[2 * l + 1]
        args = (x, H0[l], C0[l], m.wx[l], m.wh[l], m.bias[l], nx.weight, nx.bias, nh.weight, nh.bias)
        save = grad and any(t.requires_grad for t in args)
        if torch.compiler.is_compiling():
            x, h, c = torch_ops.lnlstm_fwd(*args, save)[:3]
        elif not save:  # nothing to differentiate: no autograd node
            x, h, c = ops.lnlstm_fwd_(*args, False)[:3]
        else:
            x, h, c = ops.LNLSTMFunction.apply(*args, save)
        hs.append(h)
        cs.append(c)
        if m.use_dropout and l != m.num_layers - 1:
            x = m.dropout(x)
    return x, [torch.stack(hs, 0), torch.stack(cs, 0)]


def patched_forward(original):
    """``forward`` for the reference class: the reference's own ``_before_forward`` / ``_after_forward`` around the kernels'
    layer loop, and ``original`` for everything the kernels do not compute"""

    def forward(self, inputs, prev_state, list_next_state=True):
        if accelerated(self, inputs) and inputs.shape[0] > 0:  # the reference raises its own error for T = 0
            state = self._before_forward(inputs, prev_state)
            if _state_ok(self, state, inputs):
                x, next_state = layers(self, inputs, *state)
                return x, self._after_forward(next_state, list_next_state)
        return original(self, inputs, prev_state, list_next_state)

    forward.__b200_original__ = original
    forward.__doc__ = original.__doc__
    return forward


class LSTM(nn.Module):
    """Drop-in for ding.torch_utils.network.rnn.LSTM (``lstm_type='normal'``) with LayerNorm, on CUDA fp32 tensors.

    Parameters: ``norm.{0..2L-1}`` (the LayerNorms of x Wx and h Wh of each layer), ``wx.{l}`` (I or H, 4H), ``wh.{l}``
    (H, 4H) and ``bias`` (L, 4H), drawn uniform in +-sqrt(1/H) in the order wx[l], wh[l], bias[l] for each layer.  The gates
    of each 4H row are i, f, o, u in that order.
    """

    def __init__(self, input_size: int, hidden_size: int, num_layers: int, norm_type: Optional[str] = None,
                 dropout: float = 0.) -> None:
        super(LSTM, self).__init__()
        if norm_type != 'LN':
            raise NotImplementedError("di_engine_b200.LSTM supports norm_type='LN' only (got %r)" % (norm_type, ))
        self.input_size = input_size
        self.hidden_size = hidden_size
        self.num_layers = num_layers
        G = 4 * hidden_size
        self.norm = nn.ModuleList(nn.LayerNorm(G) for _ in range(2 * num_layers))
        dims = [input_size] + [hidden_size] * num_layers
        self.wx = nn.ParameterList(nn.Parameter(torch.zeros(dims[l], G)) for l in range(num_layers))
        self.wh = nn.ParameterList(nn.Parameter(torch.zeros(hidden_size, G)) for l in range(num_layers))
        self.bias = nn.Parameter(torch.zeros(num_layers, G))
        self.use_dropout = dropout > 0.
        if self.use_dropout:
            self.dropout = nn.Dropout(dropout)
        bound = math.sqrt(1. / hidden_size)
        with torch.no_grad():
            for l in range(num_layers):
                self.wx[l].uniform_(-bound, bound)
                self.wh[l].uniform_(-bound, bound)
                self.bias[l].uniform_(-bound, bound)

    def _before_forward(self, inputs: torch.Tensor, prev_state) -> List[torch.Tensor]:
        """prev_state -> [h0, c0], each (L, B, H).  None is zeros; a list holds one entry per sample, each None (zeros), a
        dict of h and c (1 x ... in their order) or an (h, c) pair, concatenated along the batch; a dict holds h and c."""
        B = inputs.shape[1]
        if prev_state is None:
            zeros = inputs.new_zeros(self.num_layers, B, self.hidden_size)
            return [zeros, zeros]
        if isinstance(prev_state, (list, tuple)):
            if len(prev_state) != B:
                raise RuntimeError("prev_state number is not equal to batch_size: {}/{}".format(len(prev_state), B))
            zeros = inputs.new_zeros(self.num_layers, 1, self.hidden_size)
            per = [(zeros, zeros) if p is None else (tuple(p.values()) if isinstance(p, dict) else p) for p in prev_state]
            return [torch.cat(t, dim=1) for t in zip(*per)]
        if isinstance(prev_state, dict):
            return list(prev_state.values())
        raise TypeError("not support prev_state type: {}".format(type(prev_state)))

    def _after_forward(self, next_state: List[torch.Tensor],
                       list_next_state: bool = False) -> Union[List[Dict[str, torch.Tensor]], Dict[str, torch.Tensor]]:
        """[h, c] (L, B, H) -> B dicts of (L, 1, H) views when ``list_next_state``, else one dict"""
        h, c = next_state
        if not list_next_state:
            return {'h': h, 'c': c}
        B = h.shape[1]
        return [{'h': hb, 'c': cb} for hb, cb in zip(torch.chunk(h, B, dim=1), torch.chunk(c, B, dim=1))]

    def forward(self, inputs: torch.Tensor, prev_state,
                list_next_state: bool = True) -> Tuple[torch.Tensor, Union[Dict[str, torch.Tensor], list]]:
        """inputs (T, B, I) -> (output (T, B, H), next state in the form ``list_next_state`` selects)"""
        if not accelerated(self, inputs):
            raise TypeError("di_engine_b200.LSTM runs on CUDA fp32 inputs and weights only (got %s on %s)" %
                            (getattr(inputs, 'dtype', type(inputs).__name__), getattr(inputs, 'device', '?')))
        state = self._before_forward(inputs, prev_state)
        if not _state_ok(self, state, inputs):
            raise TypeError("di_engine_b200.LSTM: prev_state must hold fp32 (num_layers, batch, hidden) tensors "
                            "on the input's device")
        x, next_state = layers(self, inputs, *state)
        return x, self._after_forward(next_state, list_next_state)
