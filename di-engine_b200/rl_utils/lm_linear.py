"""GRPO, RLOO and the per-token log-probability from the lm_head's hidden states, so that the (B, S, V) logits are never
materialised.  ``hidden`` (B, S, D) and ``lm_weight`` (V, D) -- the ``nn.Linear(D, V, bias=False)`` layout of Llama,
Qwen and GPT-2 lm_heads -- are both fp32 or both bf16.  The logits exist one chunk of token rows at a time (cuBLAS
through ``torch.mm``, with the caller's matmul precision settings, as ``F.linear``); the row work runs in place on that
chunk in csrc/vocab.cu and also writes d loss / d logits, which two more GEMMs turn into d hidden and d lm_weight, each
only if its input requires grad (a frozen lm_head pays for no dW GEMM).  dW is accumulated over the chunks in fp32 and
rounded once.

These are composites, not names of ding.rl_utils:

- ``token_logp_linear(hidden, lm_weight, index)`` equals ``efficient_method(F.linear(hidden, lm_weight), index)``.  Under
  ``torch.no_grad()`` it is how a learner computes ``logp_old`` at rollout and ``logp_ref`` from the frozen reference
  model; that call allocates no gradient buffer.
- ``grpo_policy_error_linear(grpo_linear_data(...), clip_ratio, beta)`` equals ``grpo_policy_error`` on
  ``F.linear(hidden, lm_weight)`` with ``logp_old = efficient_method(logit_old, action)`` and likewise for ``logp_ref``.
- ``rloo_policy_error_linear(rloo_linear_data(...), clip_ratio)`` likewise for ``rloo_policy_error``.

``weight`` is the reference's per-token mask.  ``logp_old``, ``logp_ref``, ``adv``, ``reward`` and ``weight`` of any float
dtype are read as fp32.  Under ``torch.compile`` these functions run eagerly behind a graph break."""
from collections import namedtuple
from typing import Tuple

import torch

from .. import ops
from . import _lm_policy
from . import ppo as _ppo
from .grpo import grpo_info
from .rloo import rloo_info

grpo_linear_data = namedtuple('grpo_linear_data',
                              ['hidden', 'lm_weight', 'logp_old', 'logp_ref', 'action', 'adv', 'weight'])
rloo_linear_data = namedtuple('rloo_linear_data', ['hidden', 'lm_weight', 'logp_old', 'action', 'reward', 'weight'])


def _check_linear(hidden, lm_weight):
    """-> the dtype code of csrc/vocab.cu"""
    if hidden.dim() != 3 or min(hidden.shape) == 0:
        raise RuntimeError("hidden must be a non-empty (B, S, D), got %s" % (tuple(hidden.shape), ))
    if lm_weight.dim() != 2 or lm_weight.shape[0] == 0 or lm_weight.shape[1] != hidden.shape[2]:
        raise RuntimeError("lm_weight must be (V, D) with D = hidden's %d, got %s" %
                           (hidden.shape[2], tuple(lm_weight.shape)))
    if hidden.dtype not in ops._LOGIT_DTYPES or lm_weight.dtype != hidden.dtype:
        raise TypeError("di_engine_b200: hidden and lm_weight must both be float32 or both bfloat16 (got %s and %s)" %
                        (hidden.dtype, lm_weight.dtype))
    return ops._LOGIT_DTYPES[hidden.dtype]


def _stage(hidden, lm_weight, dev):
    """hidden as (B*S, D) and lm_weight, contiguous on ``dev`` (differentiably: autograd maps the gradients back)"""
    h = ops.to_device(hidden, dev)
    return h.reshape(-1, h.shape[-1]).contiguous(), ops.to_device(lm_weight, dev).contiguous()


def _wants_grad(h, w):
    return torch.is_grad_enabled() and (h.requires_grad or w.requires_grad)


@torch.compiler.disable
def token_logp_linear(hidden: torch.Tensor, lm_weight: torch.Tensor, index: torch.Tensor) -> torch.Tensor:
    """log softmax(hidden @ lm_weight^T)[index]: hidden (B, S, D), lm_weight (V, D), index (B, S) -> fp32 (B, S),
    differentiable w.r.t. hidden and lm_weight."""
    dt = _check_linear(hidden, lm_weight)
    B, S, _ = hidden.shape
    V = lm_weight.shape[0]
    if tuple(index.shape) != (B, S):
        raise RuntimeError("index must be (B, S) = %s, got %s" % ((B, S), tuple(index.shape)))
    dev = ops.compute_device(hidden, lm_weight, index)
    host_out = not hidden.is_cuda
    h, w = _stage(hidden, lm_weight, dev)
    a = ops.i64c(ops.to_device(index, dev), V, 'index').reshape(-1)
    if _wants_grad(h, w):
        lp = ops.TokenLogpLinearFunction.apply(h, w, a, dt)
    else:
        lp = ops.lm_logp_fwd_(h.detach(), w.detach(), a, dt)[0]
    lp = lp.view(B, S)
    return lp.cpu() if host_out else lp


def _run(kind, hidden, lm_weight, lps, action, weight, side, clip_ratio, beta, info_type):
    """the shared body of the two losses: lps = (logp_old[, logp_ref]); side ('adv', adv) or ('reward', reward)"""
    dt = _check_linear(hidden, lm_weight)
    B, S, _ = hidden.shape
    V = lm_weight.shape[0]
    _lm_policy.check_tokens(B, S, action, weight, side)
    for name, t in zip(('logp_old', 'logp_ref'), lps):
        if tuple(t.shape) != (B, S):
            raise RuntimeError("%s must be (B, S) = %s, got %s" % (name, (B, S), tuple(t.shape)))
    dev = ops.compute_device(hidden, lm_weight)
    host_out = not hidden.is_cuda
    # weight / adv / reward / the log-probabilities are read as fp32 whatever their dtype
    w = None if weight is None else ops.to_device(weight.detach(), dev).float().contiguous().reshape(-1)
    side_t = ops.to_device(side[1].detach(), dev).float().contiguous()
    side_t = side_t.reshape(side_t.shape[0], -1) if side[0] == 'reward' else side_t.reshape(-1)
    lp = [ops.to_device(t.detach(), dev).float().contiguous().reshape(-1) for t in lps]
    lp_ref = lp[1] if len(lp) > 1 else None
    a = ops.i64c(ops.to_device(action, dev), V).reshape(-1)
    h, wt = _stage(hidden, lm_weight, dev)
    cfg = (kind, B, S, dt, float(clip_ratio), float(beta))
    if _wants_grad(h, wt):
        loss, kl, cf = ops.LMLinearLossFunction.apply(h, wt, a, lp[0], lp_ref, side_t, w, *cfg)
    else:
        out = ops.lm_linear_loss_(h.detach(), wt.detach(), a, lp[0], lp_ref, side_t, w, *cfg, False, False)[0]
        loss, kl, cf = out[0], out[1], out[2]
    if host_out:
        loss = loss.cpu()
    if _ppo.LAZY_INFO:
        return loss, info_type(kl, cf)
    kl, cf = torch.stack([kl, cf]).tolist()  # one host sync
    return loss, info_type(kl, cf)


@torch.compiler.disable
def grpo_policy_error_linear(data: namedtuple, clip_ratio: float = 0.2, beta: float = 0.1) -> Tuple[torch.Tensor, namedtuple]:
    """``grpo_policy_error`` (rl_utils/grpo.py) on logits = hidden @ lm_weight^T, computed chunk by chunk.  data =
    grpo_linear_data(hidden (B, S, D), lm_weight (V, D), logp_old (B, S), logp_ref (B, S), action (B, S), adv (B),
    weight (B, S) or None).  Returns (loss, grpo_info(approx_kl, clipfrac))."""
    return _run('grpo', data.hidden, data.lm_weight, (data.logp_old, data.logp_ref), data.action, data.weight,
                ('adv', data.adv), clip_ratio, beta, grpo_info)


@torch.compiler.disable
def rloo_policy_error_linear(data: namedtuple, clip_ratio: float = 0.2) -> Tuple[torch.Tensor, namedtuple]:
    """``rloo_policy_error`` (rl_utils/rloo.py) on logits = hidden @ lm_weight^T, computed chunk by chunk.  data =
    rloo_linear_data(hidden (B, S, D), lm_weight (V, D), logp_old (B, S), action (B, S), reward (K, B / K), weight
    (B, S) or None).  Returns (loss, rloo_info(approx_kl, clipfrac))."""
    return _run('rloo', data.hidden, data.lm_weight, (data.logp_old, ), data.action, data.weight,
                ('reward', data.reward), clip_ratio, 0.0, rloo_info)


__all__ = [
    'grpo_linear_data', 'rloo_linear_data', 'token_logp_linear', 'grpo_policy_error_linear', 'rloo_policy_error_linear'
]
