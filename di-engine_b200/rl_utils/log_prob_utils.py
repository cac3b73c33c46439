"""Per-token log-probabilities of the chosen tokens (ding/rl_utils/log_prob_utils.py): ``naive_method``,
``efficient_method`` and ``less_efficient_method`` compute the same value, log softmax(logits)[index], and all three run
on the one row kernel of csrc/vocab.cu -- one streaming read of the logits, no (B, S, V) ``log_softmax`` copy and no
Python loop over B.  Logits may be fp32 or bf16; the result is fp32 either way (the reference returns bf16 for bf16
logits, rounded at each step)."""
from typing import Callable

import torch
from torch import Tensor

from .. import ops, torch_ops

LogProbFunction = Callable[[Tensor, Tensor], Tensor]

_METHODS = ('naive_method', 'efficient_method', 'less_efficient_method')


def is_fused(fn) -> bool:
    """True for the three methods of this module and the reference's own: they all go to the fused GRPO / RLOO launch."""
    name = getattr(fn, '__name__', None)
    return name in _METHODS and getattr(fn, '__module__', None) in (__name__, 'ding.rl_utils.log_prob_utils')


def _token_logp(logits: Tensor, index: Tensor) -> Tensor:
    if logits.dim() < 1 or tuple(index.shape) != tuple(logits.shape[:-1]):
        raise RuntimeError("index shape %s must equal logits shape %s without its last dimension" %
                           (tuple(index.shape), tuple(logits.shape)))
    dt = ops.logit_dtype(logits)
    dev = ops.compute_device(logits, index)
    host_out = not logits.is_cuda
    V = logits.shape[-1]
    x = ops.to_device(logits, dev)
    a = ops.i64c(ops.to_device(index, dev), V, 'index').view(-1)
    if torch.compiler.is_compiling():  # the custom op makes the kernel's 16-byte-aligned copy itself
        lp = torch_ops.token_logp(x.contiguous().view(-1, V), a)
    else:
        lp = ops.TokenLogProbFunction.apply(ops.logits_c(x).view(-1, V), a, dt)
    lp = lp.view(index.shape)
    return lp.cpu() if host_out else lp


def naive_method(logits: Tensor, index: Tensor) -> Tensor:
    """log softmax(logits)[index]: logits (B, S, V) or (S, V), index (B, S) or (S) -> fp32 (B, S) or (S)."""
    return _token_logp(logits, index)


def efficient_method(logits: Tensor, index: Tensor) -> Tensor:
    """The same value as ``naive_method`` (the reference's form gathers then subtracts logsumexp)."""
    return _token_logp(logits, index)


def less_efficient_method(logits: Tensor, index: Tensor) -> Tensor:
    """The same value as ``naive_method`` (the reference's form is ``Categorical(logits=logits).log_prob(index)``)."""
    return _token_logp(logits, index)


__all__ = ['naive_method', 'efficient_method', 'less_efficient_method', 'LogProbFunction']
