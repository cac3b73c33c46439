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

- ``ppo_policy_error_linear(ppo_policy_linear_data(...), clip_ratio, dual_clip, entropy_bonus, kl_type, entropy_weight,
  kl_weight)`` equals ``ppo_policy_error`` on ``F.linear(hidden, lm_weight)`` with ``logp_old = efficient_method(logit_old,
  action)`` and likewise for ``logp_pretrained``.
- ``a2c_error_linear(a2c_linear_data(...), value_weight, entropy_weight)`` likewise for ``a2c_error``; the gradient also
  reaches ``value``.

``weight`` is the reference's per-token mask.  ``logp_old``, ``logp_ref``, ``logp_pretrained``, ``adv``, ``reward``,
``return_``, ``value`` and ``weight`` of any float dtype are read as fp32.

Under ``torch.compile`` each call traces as one ``b200rl`` custom op (torch_ops.py) whose body is the same chunk loop, so a
learner step that ends in one of these losses compiles with ``fullgraph=True``.  The gradient rule is eager's: the forward
op writes dH / dW / d value for a unit upstream gradient, and the backward op scales them by the actual one -- out of place,
since a backward op may not return its forward's buffer (same bits as the in-place scale).  So during the backward the
saved and the scaled dW coexist: 2 x 1.09 GB at Qwen2-7B's lm_head in bf16, below the forward's own peak (the fp32
accumulator plus the rounded dW); in fp32, where eager's dW is the accumulator itself, the backward holds one (V, D)
fp32 copy more than eager's, which at D = 4096, V = 32 768 still stayed below the forward's peak (README).  A
repeated backward rescales the saved unit gradients instead of recomputing them.  ``token_logp_linear``'s backward op
recomputes each chunk's logits, as in eager mode.

PPO and A2C return their loss mix as one differentiable ``loss`` -- ``policy_loss - entropy_weight * entropy_loss +
kl_weight * kl_div``, or ``policy_loss + value_weight * value_loss - entropy_weight * entropy_loss`` -- and the components
as detached 0-dim tensors for logging, rather than three separately differentiable outputs.  The forward writes dH / dW
(and A2C's d value) for a unit upstream gradient of ``loss``, and the backward scales them in place on the device; in
eager mode a repeated backward recomputes them.  Any other mix of the components would need the logits again, which are gone after
each chunk's dW GEMM: dW = sum over chunks of dZ^T H cannot be re-weighted afterwards without one (V, D) fp32
accumulator per component (2.2 GB each at Qwen2-7B's lm_head), or a host read of the upstream gradients (a sync in the
backward).  So the weights of the mix are arguments.  A learner that wants ``ppo_error`` adds ``ppo_value_error`` on its
value head's (B, S) output to this ``loss``."""
from collections import namedtuple
from typing import Optional, Tuple

import torch

from .. import ops, torch_ops
from . import _lm_policy
from . import ppo as _ppo
from .grpo import grpo_info
from .ppo import ppo_info
from .rloo import rloo_info

grpo_linear_data = namedtuple('grpo_linear_data',
                              ['hidden', 'lm_weight', 'logp_old', 'logp_ref', 'action', 'adv', 'weight'])
rloo_linear_data = namedtuple('rloo_linear_data', ['hidden', 'lm_weight', 'logp_old', 'action', 'reward', 'weight'])
ppo_policy_linear_data = namedtuple('ppo_policy_linear_data',
                                    ['hidden', 'lm_weight', 'logp_old', 'action', 'adv', 'weight', 'logp_pretrained'])
ppo_linear_loss = namedtuple('ppo_linear_loss', ['loss', 'policy_loss', 'entropy_loss', 'kl_div'])
a2c_linear_data = namedtuple('a2c_linear_data', ['hidden', 'lm_weight', 'action', 'value', 'adv', 'return_', 'weight'])
a2c_linear_loss = namedtuple('a2c_linear_loss', ['loss', 'policy_loss', 'value_loss', 'entropy_loss'])


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
    lp = torch_ops.lm_logp(h, w, a, dt).view(B, S)
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
    loss, kl, cf = torch_ops.lm_linear_loss(h, wt, a, lp[0], lp_ref, side_t, w, *cfg)
    if host_out:
        loss = loss.cpu()
    if torch.compiler.is_compiling():  # the host read a traced graph can take, as the logit-form losses make it
        return loss, info_type(kl, cf) if _ppo.LAZY_INFO else info_type(kl.item(), cf.item())
    if _ppo.LAZY_INFO:
        return loss, info_type(kl, cf)
    kl, cf = torch.stack([kl, cf]).tolist()  # one host sync
    return loss, info_type(kl, cf)


def grpo_policy_error_linear(data: namedtuple, clip_ratio: float = 0.2, beta: float = 0.1) -> Tuple[torch.Tensor, namedtuple]:
    """``grpo_policy_error`` (rl_utils/grpo.py) on logits = hidden @ lm_weight^T, computed chunk by chunk.  data =
    grpo_linear_data(hidden (B, S, D), lm_weight (V, D), logp_old (B, S), logp_ref (B, S), action (B, S), adv (B),
    weight (B, S) or None).  Returns (loss, grpo_info(approx_kl, clipfrac))."""
    return _run('grpo', data.hidden, data.lm_weight, (data.logp_old, data.logp_ref), data.action, data.weight,
                ('adv', data.adv), clip_ratio, beta, grpo_info)


def rloo_policy_error_linear(data: namedtuple, clip_ratio: float = 0.2) -> Tuple[torch.Tensor, namedtuple]:
    """``rloo_policy_error`` (rl_utils/rloo.py) on logits = hidden @ lm_weight^T, computed chunk by chunk.  data =
    rloo_linear_data(hidden (B, S, D), lm_weight (V, D), logp_old (B, S), action (B, S), reward (K, B / K), weight
    (B, S) or None).  Returns (loss, rloo_info(approx_kl, clipfrac))."""
    return _run('rloo', data.hidden, data.lm_weight, (data.logp_old, ), data.action, data.weight,
                ('reward', data.reward), clip_ratio, 0.0, rloo_info)


def _run_pg(kind, hidden, lm_weight, action, weight, rows, value, cfg):
    """the shared body of the PPO and A2C losses: rows = the per-token (B, S) operands by name (adv, and logp_old /
    logp_pretrained or return_), value (B, S) (A2C, differentiable) or None.  -> (the one loss, the raw sums)"""
    dt = _check_linear(hidden, lm_weight)
    B, S, _ = hidden.shape
    V = lm_weight.shape[0]
    for name, t in [('action', action), ('weight', weight)] + list(rows.items()) + [('value', value)]:
        if t is not None and tuple(t.shape) != (B, S):  # check_tokens' message
            raise RuntimeError("%s must be (B, S) = %s, got %s" % (name, (B, S), tuple(t.shape)))
    dev = ops.compute_device(hidden, lm_weight)
    host_out = not hidden.is_cuda
    # the per-token operands are read as fp32 whatever their dtype; value keeps its graph (autograd casts its gradient)
    f = {k: None if t is None else ops.to_device(t.detach(), dev).float().contiguous().reshape(-1) for k, t in rows.items()}
    w = None if weight is None else ops.to_device(weight.detach(), dev).float().contiguous().reshape(-1)
    v = None if value is None else ops.to_device(value, dev).float().contiguous().reshape(-1)
    a = ops.i64c(ops.to_device(action, dev), V).reshape(-1)
    h, wt = _stage(hidden, lm_weight, dev)
    loss, out = torch_ops.lm_linear_pg(h, wt, v, a, f['adv'], w, f.get('logp_old'), f.get('logp_pretrained'),
                                       f.get('return_'), kind, dt, cfg)
    if host_out:
        loss, out = loss.cpu(), out.cpu()
    return loss, out


def ppo_policy_error_linear(data: namedtuple, clip_ratio: float = 0.2, dual_clip: Optional[float] = None,
                            entropy_bonus: bool = True, kl_type: str = 'k1', entropy_weight: float = 0.0,
                            kl_weight: float = 0.0) -> Tuple[namedtuple, namedtuple]:
    """``ppo_policy_error`` (rl_utils/ppo.py) on logits = hidden @ lm_weight^T, computed chunk by chunk.  data =
    ppo_policy_linear_data(hidden (B, S, D), lm_weight (V, D), logp_old (B, S), action (B, S), adv (B, S), weight (B, S)
    or None, logp_pretrained (B, S) or None).  Returns (ppo_linear_loss(loss, policy_loss, entropy_loss, kl_div),
    ppo_info(approx_kl, clipfrac)): ``loss = policy_loss - entropy_weight * entropy_loss + kl_weight * kl_div`` is the one
    differentiable output (to hidden and lm_weight); the components are detached, entropy_loss 0 without
    ``entropy_bonus`` and kl_div 0 without ``logp_pretrained``."""
    assert dual_clip is None or dual_clip > 1.0, "dual_clip value must be greater than 1.0, but get value: {}".format(
        dual_clip
    )
    hidden, lm_weight, logp_old, action, adv, weight, logp_pre = data
    if logp_pre is not None and kl_type not in _ppo._KL_TYPES:
        raise ValueError(f"Unknown kl_type: {kl_type}")
    if entropy_weight != 0.0 and not entropy_bonus:
        raise ValueError("ppo_policy_error_linear: entropy_weight %r needs entropy_bonus=True" % (entropy_weight, ))
    if kl_weight != 0.0 and logp_pre is None:
        raise ValueError("ppo_policy_error_linear: kl_weight %r needs logp_pretrained" % (kl_weight, ))
    cfg = (float(clip_ratio), float(dual_clip) if dual_clip is not None else 0.0, _ppo._KL_TYPES.get(kl_type, 1),
           bool(entropy_bonus), -float(entropy_weight), float(kl_weight), 0.0)
    loss, out = _run_pg('ppo', hidden, lm_weight, action, weight,
                        {'adv': adv, 'logp_old': logp_old, 'logp_pretrained': logp_pre}, None, cfg)
    if _ppo.LAZY_INFO:
        info = ppo_info(out[3], out[4])
    elif torch.compiler.is_compiling():  # the host read a traced graph can take, as the logit-form losses make it
        info = ppo_info(out[3].item(), out[4].item())
    else:
        approx_kl, clipfrac = out[3:5].tolist()  # one host sync
        info = ppo_info(approx_kl, clipfrac)
    return ppo_linear_loss(loss, out[0], out[1], out[2]), info


def a2c_error_linear(data: namedtuple, value_weight: float = 0.5, entropy_weight: float = 0.01) -> namedtuple:
    """``a2c_error`` (rl_utils/a2c.py) on logits = hidden @ lm_weight^T, computed chunk by chunk.  data =
    a2c_linear_data(hidden (B, S, D), lm_weight (V, D), action (B, S), value (B, S), adv (B, S), return_ (B, S), weight
    (B, S) or None).  Returns a2c_linear_loss(loss, policy_loss, value_loss, entropy_loss): ``loss = policy_loss +
    value_weight * value_loss - entropy_weight * entropy_loss`` is the one differentiable output (to hidden, lm_weight
    and value); the components are detached."""
    hidden, lm_weight, action, value, adv, return_, weight = data
    cfg = (0.0, 0.0, 1, True, -float(entropy_weight), 0.0, float(value_weight))
    loss, out = _run_pg('a2c', hidden, lm_weight, action, weight, {'adv': adv, 'return_': return_}, value, cfg)
    return a2c_linear_loss(loss, out[0], out[1], out[2])


__all__ = [
    'grpo_linear_data', 'rloo_linear_data', 'token_logp_linear', 'grpo_policy_error_linear', 'rloo_policy_error_linear',
    'ppo_policy_linear_data', 'ppo_linear_loss', 'ppo_policy_error_linear', 'a2c_linear_data', 'a2c_linear_loss',
    'a2c_error_linear'
]
