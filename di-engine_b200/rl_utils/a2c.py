"""``a2c_error`` and ``a2c_error_continuous`` with the signatures and namedtuples of ding/rl_utils/a2c.py:6-88 -- csrc/heads.cu
(SURVEY section 8f rank 3)."""
from collections import namedtuple

import torch

from .. import ops

a2c_data = namedtuple('a2c_data', ['logit', 'action', 'value', 'adv', 'return_', 'weight'])
a2c_loss = namedtuple('a2c_loss', ['policy_loss', 'value_loss', 'entropy_loss'])


def a2c_error(data: namedtuple) -> namedtuple:
    """
    A2C loss for a discrete action space, drop-in for ding/rl_utils/a2c.py:10-44: ``policy_loss = -mean(logp(a) * adv * w)``,
    ``value_loss = mean(w * (return_ - value)^2)``, ``entropy_loss = mean(H * w)``.  logit (B, N); action (B,) int64; value,
    adv, return_, weight (B,) (weight may be None).  Three differentiable 0-dim tensors; gradients reach ``logit`` and
    ``value``.  Forward and gradients in one launch, device-verified backward.
    """
    logit, action, value, adv, return_, weight = data
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
