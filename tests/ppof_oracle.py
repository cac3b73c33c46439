"""PPOFPolicy's advantage recompute, ding/policy/ppof.py:160-210, restated line by line around the LIVE reference functions
(``gae``, ``value_transform``, ``value_inv_transform``, ``symlog``, ``inv_symlog``) -- ppof.py itself imports treetensor and
cannot be loaded here, as with ``oracle/rl_oracle.ppo_policy_gae_returns`` for policy/ppo.py.

The critic's ``compute_critic`` output is the dict ``{'pred': ...}``; the model call is replaced by the given tensors.
PopArt's ``update_parameters`` (:198) and the ``RunningMeanStd.update`` call of :208 are model / host state: the restatement
returns what :208 hands to ``update`` as (np.mean, np.var, count) over all elements instead.
"""
import numpy as np
import torch

_F = np.float32


def _sign(x):
    return (0 < x).astype(_F) - (x < 0).astype(_F)  # torch.sign: 0 for NaN and -0


def h_ieee(x):
    """value_transform with every op rounded once as IEEE fp32 (numpy's sqrt is correctly rounded; torch's vectorised CPU
    sqrt is not always -- it is 1 ulp off for some inputs -- so the live function cannot pin a kernel that rounds correctly)"""
    a = x.numpy()
    with np.errstate(all='ignore'):
        r = _sign(a) * (np.sqrt(np.abs(a) + _F(1)) - _F(1)) + _F(0.01) * a
    return torch.from_numpy(r.astype(_F))


def h_inv_ieee(x):
    """value_inv_transform, IEEE fp32 op by op (4 eps and 2 eps as the python doubles, rounded to fp32; true division)"""
    a = x.numpy()
    with np.errstate(all='ignore'):
        u = (np.sqrt(_F(1) + _F(4 * 1e-2) * ((np.abs(a) + _F(1)) + _F(1e-2))) - _F(1)) / _F(2 * 1e-2)
        r = _sign(a) * (u * u - _F(1))
    return torch.from_numpy(r.astype(_F))


def ppof_recompute(ref, pred, next_pred, reward, done, traj_flag, gamma, lambda_, value_norm, std=None, mu=None,
                   sigma=None, ieee_sqrt=False):
    """-> (adv, value, return_, return_stats or None); the inputs are cloned first (gae masks next_value in place).
    ``ieee_sqrt``: 'value_rescale' through ``h_ieee`` / ``h_inv_ieee`` instead of the live functions (CPU tensors)."""
    value_transform = h_ieee if ieee_sqrt else ref.value_transform
    value_inv_transform = h_inv_ieee if ieee_sqrt else ref.value_inv_transform
    value = {'pred': pred.clone()}
    next_value = {'pred': next_pred.clone()}
    assert value_norm in ['popart', 'value_rescale', 'symlog', 'baseline']
    if value_norm == 'popart':  # :171-180
        reward = (reward - mu) / sigma
        value = value['pred']
        next_value = next_value['pred']
    elif value_norm == 'value_rescale':  # :181-183
        value = value_inv_transform(value['pred'])
        next_value = value_inv_transform(next_value['pred'])
    elif value_norm == 'symlog':  # :184-186
        value = ref.inv_symlog(value['pred'])
        next_value = ref.inv_symlog(next_value['pred'])
    elif value_norm == 'baseline':  # :187-189
        value = value['pred'] * std
        next_value = next_value['pred'] * std
    adv_data = ref.gae_data(value, next_value, reward, done, traj_flag)  # :191-192
    adv = ref.gae(adv_data, gamma, lambda_)  # :193
    unnormalized_returns = value + adv  # :195
    stats = None
    if value_norm == 'value_rescale':  # :199-201
        value = value_transform(value)
        unnormalized_returns = value_transform(unnormalized_returns)
    elif value_norm == 'symlog':  # :202-204
        value = ref.symlog(value)
        unnormalized_returns = ref.symlog(unnormalized_returns)
    elif value_norm == 'baseline':  # :205-208
        value /= std
        unnormalized_returns /= std
        x = unnormalized_returns.cpu().numpy().reshape(-1)
        stats = (float(np.mean(x)), float(np.var(x)), float(x.shape[0]))
    return adv, value, unnormalized_returns, stats
