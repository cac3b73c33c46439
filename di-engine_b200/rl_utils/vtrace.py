"""``vtrace_error_discrete_action`` with the signature of ding/rl_utils/vtrace.py:48-49,72-79 -- csrc/pg.cu."""
from collections import namedtuple

import torch

from .. import ops, torch_ops

vtrace_data = namedtuple('vtrace_data', ['target_output', 'behaviour_output', 'action', 'value', 'reward', 'weight'])
vtrace_loss = namedtuple('vtrace_loss', ['policy_loss', 'value_loss', 'entropy_loss'])


def shape_fn_vtrace_discrete_action(args, kwargs):
    """Plugin-cache key of the reference boundary (vtrace.py:52-63): the (T, B, N) shape of ``target_output``."""
    data = args[0] if len(args) > 0 else kwargs['data']
    return data.target_output.shape


def vtrace_error_discrete_action(
    data: namedtuple,
    gamma: float = 0.99,
    lambda_: float = 0.95,
    rho_clip_ratio: float = 1.0,
    c_clip_ratio: float = 1.0,
    rho_pg_clip_ratio: float = 1.0
):
    """
    V-trace actor-critic loss (IMPALA, arXiv:1802.01561), drop-in for ding/rl_utils/vtrace.py:72-136.
    target_output, behaviour_output (T, B, N); action (T, B) int64; value (T+1, B); reward (T, B); weight None or
    (T, B).  Returns ``vtrace_loss(policy_loss, value_loss, entropy_loss)``; gradients reach ``target_output`` and
    ``value`` (row T of ``value`` gets zero, as value[:-1] in vtrace.py:134).
    """
    target_output, behaviour_output, action, value, reward, weight = data
    dev = ops.compute_device(target_output, value)
    host_out = not target_output.is_cuda
    if target_output.dim() != 3 or value.dim() != 2 or reward.dim() != 2:
        raise ValueError("expected target_output (T, B, N), value (T+1, B), reward (T, B)")
    T, B, N = target_output.shape
    if value.shape != (T + 1, B) or reward.shape != (T, B) or action.shape != (T, B) or \
            behaviour_output.shape != target_output.shape:
        raise ValueError("vtrace shapes do not match: target %s behaviour %s action %s value %s reward %s" % (
            tuple(target_output.shape), tuple(behaviour_output.shape), tuple(action.shape), tuple(value.shape),
            tuple(reward.shape)))
    tgt = ops.f32c(ops.to_device(target_output, dev), 'target_output')
    beh = ops.f32c(ops.to_device(behaviour_output.detach(), dev), 'behaviour_output')
    act = ops.i64c(ops.to_device(action, dev), target_output.shape[-1])
    v = ops.f32c(ops.to_device(value, dev), 'value')
    r = ops.f32c(ops.to_device(reward.detach(), dev), 'reward')
    w = None
    if weight is not None:
        w = ops.f32c(ops.to_device(weight.detach(), dev), 'weight')
        if w.shape != r.shape:
            w = w.expand_as(r).contiguous()
    args = (tgt, v, beh, act, r, w, float(gamma), float(lambda_), float(rho_clip_ratio), float(c_clip_ratio),
            float(rho_pg_clip_ratio))
    p, vl, e = torch_ops.vtrace(*args) if torch.compiler.is_compiling() else ops.VTraceFunction.apply(*args)
    if host_out:
        p, vl, e = p.cpu(), vl.cpu(), e.cpu()
    return vtrace_loss(p, vl, e)


def vtrace_error_continuous_action(
        data: namedtuple,
        gamma: float = 0.99,
        lambda_: float = 0.95,
        rho_clip_ratio: float = 1.0,
        c_clip_ratio: float = 1.0,
        rho_pg_clip_ratio: float = 1.0
):
    """
    V-trace (IMPALA) loss for a continuous action space, drop-in for ding/rl_utils/vtrace.py:139-212: ``target_output`` and
    ``behaviour_output`` are dicts ``{'mu': (T, B, D), 'sigma': (T, B, D)}`` of ``Independent(Normal)`` policies, action
    (T, B, D) float, value (T+1, B), reward / weight (T, B).  Returns ``vtrace_loss``; gradients reach the target policy's
    ``mu`` / ``sigma`` and ``value``.  Rows kernel -> the scan of the discrete head -> backward rows kernel (csrc/pg.cu).
    """
    target_output, behaviour_output, action, value, reward, weight = data
    mu, sigma = target_output['mu'], target_output['sigma']
    dev = ops.compute_device(mu, value)
    host_out = not mu.is_cuda
    T, B = reward.shape
    D = mu.shape[-1]
    for name, t_, n in (('mu', mu, T * B * D), ('sigma', sigma, T * B * D), ('behaviour mu', behaviour_output['mu'], T * B * D),
                        ('behaviour sigma', behaviour_output['sigma'], T * B * D), ('action', action, T * B * D),
                        ('value', value, (T + 1) * B)):
        if t_.numel() != n:
            raise ValueError("vtrace_error_continuous_action: %s %s does not match reward %s" %
                             (name, tuple(t_.shape), tuple(reward.shape)))
    f = lambda t, nm: ops.f32c(ops.to_device(t, dev), nm)  # noqa: E731
    w = f(weight.detach(), 'weight') if weight is not None else None
    p, v, e = ops.VTraceContinuousFunction.apply(
        f(mu, 'mu'), f(sigma, 'sigma'), f(value, 'value'), f(behaviour_output['mu'].detach(), 'mu_b'),
        f(behaviour_output['sigma'].detach(), 'sigma_b'), f(action.detach(), 'action'), f(reward.detach(), 'reward'), w, D,
        float(gamma), float(lambda_), float(rho_clip_ratio), float(c_clip_ratio), float(rho_pg_clip_ratio))
    if host_out:
        p, v, e = p.cpu(), v.cpu(), e.cpu()
    return vtrace_loss(p, v, e)


def impala_reshape_data(values: torch.Tensor, rewards: torch.Tensor, done: torch.Tensor):
    """
    The masking ``IMPALAPolicy._reshape_data`` applies between the model output and ``vtrace_error_*`` (ding/policy/impala.py:
    316-322) -- not a reference function, exactly those lines in one elementwise launch (csrc/policy.cu)::

        weights_ = 1 - done.float();  weights = torch.ones_like(rewards)
        values[1:] = values[1:] * weights_;  weights[1:] = weights_[:-1];  rewards = rewards * weights

    values (T+1, B) -- gradient flows back through the mask to the critic output --, rewards and done (T, B).
    Returns ``(values, rewards, weights)`` ready for ``vtrace_data(..., value=values, reward=rewards, weight=weights)``.
    Unlike the reference the input ``values`` is not modified in place.
    """
    dev = ops.compute_device(values, rewards)
    host_out = not values.is_cuda
    v = ops.f32c(ops.to_device(values, dev), 'values')
    r = ops.f32c(ops.to_device(rewards.detach(), dev), 'rewards')
    d = ops.f32c(ops.to_device(done.detach(), dev), 'done')
    if v.dim() != 2 or r.dim() != 2 or v.shape[0] != r.shape[0] + 1 or v.shape[1] != r.shape[1] or d.shape != r.shape:
        raise ValueError("expected values (T+1, B), rewards / done (T, B); got %s / %s / %s" %
                         (tuple(values.shape), tuple(rewards.shape), tuple(done.shape)))
    vo, ro, wo = ops.ImpalaMaskFunction.apply(v, r, d)
    return (vo.cpu(), ro.cpu(), wo.cpu()) if host_out else (vo, ro, wo)
