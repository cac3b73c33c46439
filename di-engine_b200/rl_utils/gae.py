"""``gae`` / ``gae_data`` with the signatures of ding/rl_utils/gae.py:5,25 -- computed by ``b200rl_gae`` (csrc/gae.cu)."""
from collections import namedtuple

import torch

from .. import ops, torch_ops

gae_data = namedtuple('gae_data', ['value', 'next_value', 'reward', 'done', 'traj_flag'])
gae_returns_out = namedtuple('gae_returns_out', ['adv', 'value', 'return_', 'unnormalized_return', 'return_stats', 'adv_stats'])


def shape_fn_gae(args, kwargs):
    """Plugin-cache key of the reference boundary (ding/rl_utils/gae.py:8-19): the (T, B) shape of ``reward``."""
    data = args[0] if len(args) > 0 else kwargs['data']
    return data.reward.shape


def gae(data: namedtuple, gamma: float = 0.99, lambda_: float = 0.97) -> torch.FloatTensor:
    """
    Generalized Advantage Estimator, drop-in for ding/rl_utils/gae.py:25-70.

    Shapes: value, next_value (T, B) -- or (T,) or (T, B, A) with (T, B) reward (gae.py:56-59); reward (T, B);
    done / traj_flag (T, B), ``None`` (-> zeros / -> done, gae.py:51-54), bool or float.  Returns adv shaped like
    ``value``.  As in the reference, ``next_value`` is masked IN PLACE by ``(1 - done)`` (gae.py:61).
    The result is bit-identical to the reference loop (same fp32 operations in the same order).
    Like the reference's callers (policy/ppo.py:279-281 under ``torch.no_grad()``) no autograd graph is built.
    """
    value, next_value, reward, done, traj_flag = data
    dev = ops.compute_device(value, next_value, reward)
    host_out = not value.is_cuda
    if value.dim() == reward.dim() + 1:
        agents = value.shape[-1]
        lead = value.shape[:-1]
    else:
        agents = 1
        lead = value.shape
    if tuple(lead) != tuple(reward.shape) or next_value.shape != value.shape:
        raise ValueError(
            "gae: value %s / next_value %s / reward %s shapes do not match" %
            (tuple(value.shape), tuple(next_value.shape), tuple(reward.shape))
        )
    v = ops.f32c(ops.to_device(value.detach(), dev), 'value')
    nv_src = next_value.detach()
    nv = ops.f32c(ops.to_device(nv_src, dev), 'next_value')
    r = ops.f32c(ops.to_device(reward.detach(), dev), 'reward')
    d = ops.f32c(ops.to_device(done.detach(), dev), 'done') if done is not None else None
    tf = ops.f32c(ops.to_device(traj_flag.detach(), dev), 'traj_flag') if traj_flag is not None else None
    if d is not None and d.shape != r.shape:
        d = d.expand_as(r).contiguous()
    if tf is not None and tf.shape != r.shape:
        tf = tf.expand_as(r).contiguous()
    if torch.compiler.is_compiling():
        adv = torch_ops.gae_op(v, nv, r, d, tf, float(gamma), float(lambda_), agents)
        staged = nv is not nv_src
    else:
        adv = ops.gae_(v, nv, r, d, tf, gamma, lambda_, agents)
        staged = nv.data_ptr() != nv_src.data_ptr()
    if d is not None and staged:
        # the kernel masked a staged / re-laid-out copy: propagate the reference's in-place side effect
        with torch.no_grad():
            next_value.copy_(nv.to(next_value.device))
    return adv.cpu() if host_out else adv


def gae_returns(data: namedtuple, gamma: float = 0.99, lambda_: float = 0.97, value_norm_std=None) -> namedtuple:
    """
    ``gae`` together with the batch-level pieces ``PPOPolicy._forward_learn`` wraps around it when it recomputes the advantage
    (ding/policy/ppo.py:274-297) -- not a reference function, exactly those reference lines in one call (csrc/policy.cu)::

        value *= std; next_value *= std                      # only with value_norm (std = RunningMeanStd.std, a float)
        adv = gae(gae_data(value, next_value, reward, done, traj_flag), gamma, lambda_)
        unnormalized_returns = value + adv
        value = value / std; return_ = unnormalized_returns / std   # value / return_ as the learner stores them
        running_mean_std.update(unnormalized_returns.cpu().numpy()) # here: three device floats {mean, np.var, count}

    ``data`` as for ``gae`` with value shaped like reward ((T,) -- the real learner: ONE sequence of n_sample steps, cut into
    independent segments at every traj_flag == 1 and scanned segment-parallel, bit-identical to the loop -- or (T, B));
    ``value_norm_std`` None (value_norm off) or the running std.  The inputs are NOT modified.  Returns
    ``gae_returns_out(adv, value, return_, unnormalized_return, return_stats)``; ``return_stats`` = (mean, population variance,
    count) of the unnormalized returns: what ``RunningMeanStd.update`` (ding/utils/default_helper.py:547-567) computes from the
    array the reference first copies to the host; ``adv_stats`` = (adv.mean(), adv.std() + 1e-8) of the whole batch, computed
    in the same pass: hand it to ``ppo_error_adv_norm(..., adv_stats=...)`` when the batch is ONE minibatch
    (policy/ppo.py:304-306 normalises per minibatch: those take their own statistics, ``ops.adv_stats_``).
    """
    value, next_value, reward, done, traj_flag = data
    dev = ops.compute_device(value, next_value, reward)
    host_out = not value.is_cuda
    if value.shape != reward.shape or next_value.shape != value.shape or value.dim() not in (1, 2):
        raise ValueError("gae_returns: value %s / next_value %s / reward %s must share a (T,) or (T, B) shape" %
                         (tuple(value.shape), tuple(next_value.shape), tuple(reward.shape)))
    v = ops.f32c(ops.to_device(value.detach(), dev), 'value')
    nv = ops.f32c(ops.to_device(next_value.detach(), dev), 'next_value')
    r = ops.f32c(ops.to_device(reward.detach(), dev), 'reward')
    d = ops.f32c(ops.to_device(done.detach(), dev), 'done') if done is not None else None
    tf = ops.f32c(ops.to_device(traj_flag.detach(), dev), 'traj_flag') if traj_flag is not None else None
    vs = 0.0 if value_norm_std is None else float(value_norm_std)
    if torch.compiler.is_compiling():
        adv, unnorm, vout, rout, stats, astats = torch_ops.gae_returns(v, nv, r, d, tf, gamma, lambda_, vs)
    else:
        adv, unnorm, vout, rout, stats, astats = ops.gae_returns_(v, nv, r, d, tf, gamma, lambda_, 1, vs, True, True,
                                                                  want_adv_stats=True)
    if vs == 0.0:
        vout, rout = v, unnorm
    out = gae_returns_out(adv, vout, rout, unnorm, stats, astats)
    return gae_returns_out(*[t.cpu() for t in out]) if host_out else out


ppof_gae_returns_out = namedtuple('ppof_gae_returns_out', ['adv', 'value', 'return_', 'return_stats', 'adv_stats'])


def ppof_gae_returns(data: namedtuple, gamma: float = 0.99, lambda_: float = 0.97, value_norm: str = 'baseline', std=None,
                     popart_mu=None, popart_sigma=None) -> namedtuple:
    """
    ``PPOFPolicy.forward``'s advantage recompute (ding/policy/ppof.py:160-210) in one call -- not a reference function, exactly
    those reference lines (csrc/policy.cu)::

        # decode the critic's output ('pred') -- ppof.py:171-189
        popart:        reward = (reward - mu) / sigma            value, next_value as they are
        value_rescale: value = value_inv_transform(value)        next_value likewise
        symlog:        value = inv_symlog(value)                 next_value likewise
        baseline:      value = value * std                       next_value likewise   (std = RunningMeanStd.std)
        adv = gae(gae_data(value, next_value, reward, done, traj_flag), gamma, lambda_)
        unnormalized_returns = value + adv
        # encode -- ppof.py:197-210
        value_rescale: value, return_ = value_transform(value), value_transform(unnormalized_returns)
        symlog:        value, return_ = symlog(value), symlog(unnormalized_returns)
        baseline:      value, return_ = value / std, unnormalized_returns / std
                       running_mean_std.update(return_.cpu().numpy())   # here: three device floats {mean, np.var, count}
        popart:        value, return_ = value, unnormalized_returns

    ``data`` as for ``gae``: value shaped like reward ((n,) -- PPOF's one sequence of n_sample steps, scanned in one launch --
    or (T, B)), or with a trailing dim of 1 against that reward (PopArt's (n, 1) prediction, gae.py:56-59).  ``std``: the
    running std, required for 'baseline'.  ``popart_mu`` / ``popart_sigma``: the PopArt head's ``mu`` / ``sigma`` buffers
    (one float each, read on the device), required for 'popart'.  The inputs are NOT modified (the reference masks
    ``next_value`` in place inside ``gae``).  Returns ``ppof_gae_returns_out(adv, value, return_, return_stats, adv_stats)``
    with adv / value / return_ shaped like value; ``return_stats`` = (mean, population variance, count) of ``return_`` in
    'baseline' (what ``RunningMeanStd.update`` computes from it), None otherwise; ``adv_stats`` = (adv.mean(), adv.std() + 1e-8)
    of the whole batch from the same pass.  PopArt's ``update_parameters`` and ``RunningMeanStd.update`` stay with the caller.
    """
    value, next_value, reward, done, traj_flag = data
    if value_norm not in ops.VALUE_NORMS:
        raise ValueError("ppof_gae_returns: value_norm must be one of %s, got %r" % (ops.VALUE_NORMS, value_norm))
    if value_norm == 'baseline':
        if std is None:
            raise ValueError("ppof_gae_returns: value_norm='baseline' needs std (RunningMeanStd.std)")
        std = float(std)
        if not std > 0.0:
            raise ValueError("ppof_gae_returns: std must be > 0, got %r" % std)
    else:
        std = 0.0
    if value_norm == 'popart' and (popart_mu is None or popart_sigma is None):
        raise ValueError("ppof_gae_returns: value_norm='popart' needs popart_mu and popart_sigma")
    lead = value.shape[:-1] if (value.dim() == reward.dim() + 1 and value.shape[-1] == 1) else value.shape
    if tuple(lead) != tuple(reward.shape) or next_value.shape != value.shape or reward.dim() not in (1, 2):
        raise ValueError("ppof_gae_returns: value %s / next_value %s / reward %s must share a (T,) or (T, B) shape" %
                         (tuple(value.shape), tuple(next_value.shape), tuple(reward.shape)))
    dev = ops.compute_device(value, next_value, reward)
    host_out = not value.is_cuda
    v = ops.f32c(ops.to_device(value.detach(), dev), 'value').reshape(reward.shape)
    nv = ops.f32c(ops.to_device(next_value.detach(), dev), 'next_value').reshape(reward.shape)
    r = ops.f32c(ops.to_device(reward.detach(), dev), 'reward')
    d = ops.f32c(ops.to_device(done.detach(), dev), 'done') if done is not None else None
    tf = ops.f32c(ops.to_device(traj_flag.detach(), dev), 'traj_flag') if traj_flag is not None else None
    if d is not None and d.shape != r.shape:
        d = d.expand_as(r).contiguous()
    if tf is not None and tf.shape != r.shape:
        tf = tf.expand_as(r).contiguous()
    mu = sigma = None
    if value_norm == 'popart':
        mu = ops.f32c(ops.to_device(popart_mu.detach(), dev), 'popart_mu').reshape(-1)
        sigma = ops.f32c(ops.to_device(popart_sigma.detach(), dev), 'popart_sigma').reshape(-1)
        if mu.numel() != 1 or sigma.numel() != 1:
            raise ValueError("ppof_gae_returns: popart_mu / popart_sigma must hold one float each (a single-output PopArt head)")
    if torch.compiler.is_compiling():
        adv, vout, rout, stats, astats = torch_ops.ppof_gae_returns(v, nv, r, d, tf, gamma, lambda_, value_norm, std, mu,
                                                                    sigma)
    else:
        adv, vout, rout, stats, astats = ops.gae_returns_norm_(v, nv, r, d, tf, gamma, lambda_, value_norm, std, mu, sigma,
                                                               value_norm == 'baseline')
    out = ppof_gae_returns_out(adv.reshape(value.shape), vout.reshape(value.shape), rout.reshape(value.shape), stats, astats)
    if host_out:
        out = ppof_gae_returns_out(*[None if t is None else t.cpu() for t in out])
    return out
