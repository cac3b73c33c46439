"""``a2c_error`` and ``a2c_error_continuous`` with the signatures and namedtuples of ding/rl_utils/a2c.py:6-88 -- csrc/heads.cu
(SURVEY section 8f rank 3); language-model calls of ``a2c_error`` (bf16 logits, or fp32 with V >= ``ppo.LM_MIN_VOCAB``) run
on the vocabulary-scale row kernel of csrc/vocab.cu."""
from collections import namedtuple

import torch

from .. import ops, torch_ops
from . import ppo as _ppo

a2c_data = namedtuple('a2c_data', ['logit', 'action', 'value', 'adv', 'return_', 'weight'])
a2c_loss = namedtuple('a2c_loss', ['policy_loss', 'value_loss', 'entropy_loss'])


def a2c_error(data: namedtuple) -> namedtuple:
    """
    A2C loss for a discrete action space, drop-in for ding/rl_utils/a2c.py:10-44: ``policy_loss = -mean(logp(a) * adv * w)``,
    ``value_loss = mean(w * (return_ - value)^2)``, ``entropy_loss = mean(H * w)``.  logit (B, N); action (B,) int64; value,
    adv, return_, weight (B,) (weight may be None).  Three differentiable 0-dim tensors; gradients reach ``logit`` and
    ``value``.  Forward and gradients in one launch, device-verified backward.

    Language-model shapes -- logits (..., V), e.g. (B, S, V) against (B, S) action / value / adv / return_ / weight, in
    bf16 or in fp32 with V >= ``ppo.LM_MIN_VOCAB`` -- run on the vocabulary-scale row kernel of csrc/vocab.cu.
    """
    logit, action, value, adv, return_, weight = data
    if _ppo._lm_path(logit, adv):
        return _a2c_lm(logit, action, value, adv, return_, weight)
    dev = ops.compute_device(logit, value)
    host_out = not logit.is_cuda
    N = logit.shape[-1]
    S = logit.numel() // N
    for name, t_ in (('action', action), ('value', value), ('adv', adv), ('return_', return_), ('weight', weight)):
        if t_ is not None and t_.numel() != S:
            raise ValueError("a2c_error: %s %s does not match logit %s" % (name, tuple(t_.shape), tuple(logit.shape)))
    z = ops.f32c(ops.to_device(logit, dev), 'logit')
    v = ops.f32c(ops.to_device(value, dev), 'value')
    a = ops.i64c(ops.to_device(action, dev), logit.shape[-1])
    ad = ops.f32c(ops.to_device(adv.detach(), dev), 'adv')
    rt = ops.f32c(ops.to_device(return_.detach(), dev), 'return_')
    w = ops.f32c(ops.to_device(weight.detach(), dev), 'weight') if weight is not None else None
    p, vl, e = ops.A2CFunction.apply(z, v, a, ad, rt, w, S, N)
    if host_out:
        p, vl, e = p.cpu(), vl.cpu(), e.cpu()
    return a2c_loss(p, vl, e)


def _a2c_lm(logit, action, value, adv, return_, weight):
    """a2c_error on token rows (csrc/vocab.cu, ops.A2CLMFunction): the reference's plain means over all rows, under the
    call site's existing ``'a2c'`` expected-upstream-gradient record"""
    dt = ops.logit_dtype(logit)
    V = logit.shape[-1]
    rows = logit.numel() // V
    for name, t_ in (('action', action), ('value', value), ('adv', adv), ('return_', return_), ('weight', weight)):
        if t_ is not None and t_.numel() != rows:
            raise ValueError("a2c_error: %s %s does not match logit %s" % (name, tuple(t_.shape), tuple(logit.shape)))
    if value.dtype not in (torch.float32, torch.bfloat16):
        raise TypeError("di_engine_b200: a2c_error on language-model logits takes a float32 or bfloat16 value (got %s)" %
                        value.dtype)
    dev = ops.compute_device(logit, value)
    host_out = not logit.is_cuda
    compiling = torch.compiler.is_compiling()
    # a traced tensor has no address: the custom op makes the kernel's 16-byte-aligned copy itself
    z = ops.to_device(logit, dev).contiguous() if compiling else ops.logits_c(ops.to_device(logit, dev))
    # a bf16 value is read as fp32; autograd's cast hands its gradient back in bf16
    v = ops.to_device(value, dev).float().contiguous()
    a = ops.i64c(ops.to_device(action, dev), V)
    ad, rt = (ops.to_device(t_.detach(), dev).float().contiguous() for t_ in (adv, return_))
    w = ops.to_device(weight.detach(), dev).float().contiguous() if weight is not None else None
    p, vl, e = torch_ops.a2c_lm(z, v, a, ad, rt, w) if compiling else ops.A2CLMFunction.apply(z, v, a, ad, rt, w, dt)
    if host_out:
        p, vl, e = p.cpu(), vl.cpu(), e.cpu()
    return a2c_loss(p, vl, e)


def a2c_error_continuous(data: namedtuple) -> namedtuple:
    """
    A2C loss for a continuous action space, drop-in for ding/rl_utils/a2c.py:50-88: the policy is
    ``Independent(Normal(mu, sigma), 1)`` given as the dict ``logit = {'mu': (B, D), 'sigma': (B, D)}``; action (B, D) float;
    value, adv, return_, weight (B,) (weight may be None).  The three losses of ``a2c_error``; gradients reach ``mu``,
    ``sigma`` and ``value`` (``action`` is taken detached).  Forward and gradients in one launch, device-verified backward.
    """
    logit, action, value, adv, return_, weight = data
    mu, sigma = logit['mu'], logit['sigma']
    dev = ops.compute_device(mu, value)
    host_out = not mu.is_cuda
    D = mu.shape[-1] if mu.dim() else 1
    S = mu.numel() // D
    for name, t_, n in (('sigma', sigma, S * D), ('action', action, S * D), ('value', value, S), ('adv', adv, S),
                        ('return_', return_, S), ('weight', weight, S)):
        if t_ is not None and t_.numel() != n:
            raise ValueError("a2c_error_continuous: %s %s does not match mu %s" % (name, tuple(t_.shape), tuple(mu.shape)))
    m = ops.f32c(ops.to_device(mu, dev), 'mu')
    sg = ops.f32c(ops.to_device(sigma, dev), 'sigma')
    v = ops.f32c(ops.to_device(value, dev), 'value')
    ac = ops.f32c(ops.to_device(action.detach(), dev), 'action')
    ad = ops.f32c(ops.to_device(adv.detach(), dev), 'adv')
    rt = ops.f32c(ops.to_device(return_.detach(), dev), 'return_')
    w = ops.f32c(ops.to_device(weight.detach(), dev), 'weight') if weight is not None else None
    p, vl, e = ops.A2CContinuousFunction.apply(m, sg, v, ac, ad, rt, w, S, D)
    if host_out:
        p, vl, e = p.cpu(), vl.cpu(), e.cpu()
    return a2c_loss(p, vl, e)
