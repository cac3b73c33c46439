"""``happo_error`` / ``happo_policy_error`` / ``happo_value_error`` with the signatures of ding/rl_utils/happo.py:18,81,150 -- the
PPO kernels (csrc/ppo.cu) with the per-sample ``factor`` operand: ``min(surr1, surr2) * factor`` before the dual clip."""
from collections import namedtuple
from typing import Optional, Tuple

import torch

from .ppo import (_ppo_error, _ppo_error_continuous, ppo_data, ppo_value_data, ppo_value_error)

happo_value_data = namedtuple('happo_value_data', ['value_new', 'value_old', 'return_', 'weight'])
happo_loss = namedtuple('happo_loss', ['policy_loss', 'value_loss', 'entropy_loss'])
happo_policy_loss = namedtuple('happo_policy_loss', ['policy_loss', 'entropy_loss'])
happo_info = namedtuple('happo_info', ['approx_kl', 'clipfrac'])
happo_data = namedtuple(
    'happo_data', ['logit_new', 'logit_old', 'action', 'value_new', 'value_old', 'adv', 'return_', 'weight', 'factor']
)
happo_policy_data = namedtuple('happo_policy_data', ['logit_new', 'logit_old', 'action', 'adv', 'weight', 'factor'])


def happo_error(
        data: namedtuple,
        clip_ratio: float = 0.2,
        use_value_clip: bool = True,
        dual_clip: Optional[float] = None,
) -> Tuple[namedtuple, namedtuple]:
    """
    Drop-in for ding/rl_utils/happo.py:18-78: logit_new / logit_old (B, N), action (B,), value_new / value_old / adv / return_
    (B,), weight None or (B,), factor (B, 1).  Returns ``(happo_loss(policy_loss, value_loss, entropy_loss), happo_info)``; the
    losses are attached to ``logit_new`` and ``value_new``.  One launch forward (+ gradients), device-verified backward, as
    ``ppo_error``; its expected-upstream-gradient record is kept apart from the PPO ones.
    """
    logit_new, logit_old, action, value_new, value_old, adv, return_, weight, factor = data
    loss, info = _ppo_error(
        ppo_data(logit_new, logit_old, action, value_new, value_old, adv, return_, weight, None), clip_ratio, use_value_clip,
        dual_clip, 'k1', 'happo', factor=factor
    )
    return happo_loss(loss.policy_loss, loss.value_loss, loss.entropy_loss), happo_info(info.approx_kl, info.clipfrac)


def happo_policy_error(
        data: namedtuple,
        clip_ratio: float = 0.2,
        dual_clip: Optional[float] = None,
) -> Tuple[namedtuple, namedtuple]:
    """Drop-in for ding/rl_utils/happo.py:81-147 (the policy half: zero value head, as ``ppo_policy_error``)."""
    assert dual_clip is None or dual_clip > 1.0, "dual_clip value must be greater than 1.0, but get value: {}".format(
        dual_clip
    )
    logit_new, logit_old, action, adv, weight, factor = data
    zero = torch.zeros_like(adv)
    loss, info = _ppo_error(
        ppo_data(logit_new, logit_old, action, zero, zero, adv, zero, weight, None), clip_ratio, False, dual_clip, 'k1',
        'happo_policy', factor=factor
    )
    return happo_policy_loss(loss.policy_loss, loss.entropy_loss), happo_info(info.approx_kl, info.clipfrac)


def happo_value_error(
        data: namedtuple,
        clip_ratio: float = 0.2,
        use_value_clip: bool = True,
) -> torch.Tensor:
    """Drop-in for ding/rl_utils/happo.py:150-192 -- the same expression as ``ppo_value_error`` (ppo.py:233-275)."""
    value_new, value_old, return_, weight = data
    return ppo_value_error(ppo_value_data(value_new, value_old, return_, weight), clip_ratio, use_value_clip)


def happo_error_continuous(
        data: namedtuple,
        clip_ratio: float = 0.2,
        use_value_clip: bool = True,
        dual_clip: Optional[float] = None,
) -> Tuple[namedtuple, namedtuple]:
    """
    Drop-in for ding/rl_utils/happo.py:195-284: ``happo_data`` whose ``logit_new`` / ``logit_old`` fields are dicts
    ``{'mu': (B, D), 'sigma': (B, D)}``; action (B, D); factor (B, 1).  Differences to ``ppo_error_continuous`` as in the
    reference: ``factor * min(surr1, surr2)`` before the dual clip, entropy and approx_kl averaged over the B * D per-dimension
    terms (``Normal`` instead of ``Independent(Normal)``).  The continuous-PPO kernel with its factor operand (csrc/heads.cu).
    """
    mu_sigma_new, mu_sigma_old, action, value_new, value_old, adv, return_, weight, factor = data
    loss, info = _ppo_error_continuous(
        ppo_data(mu_sigma_new, mu_sigma_old, action, value_new, value_old, adv, return_, weight, None), clip_ratio,
        use_value_clip, dual_clip, 'k1', 'happoc', factor=factor
    )
    return happo_loss(loss.policy_loss, loss.value_loss, loss.entropy_loss), happo_info(info.approx_kl, info.clipfrac)


def happo_policy_error_continuous(data: namedtuple,
                                  clip_ratio: float = 0.2,
                                  dual_clip: Optional[float] = None) -> Tuple[namedtuple, namedtuple]:
    """
    Drop-in for ding/rl_utils/happo.py:287-347: five fields ``(mu_sigma_new, mu_sigma_old, action, adv, weight)`` -- the
    reference's body takes no factor here and is the policy half of ``ppo_error_continuous`` (Independent(Normal)) word for
    word; zero value head, as ``ppo_policy_error``.
    """
    mu_sigma_new, mu_sigma_old, action, adv, weight = data
    zero = torch.zeros_like(adv)
    loss, info = _ppo_error_continuous(
        ppo_data(mu_sigma_new, mu_sigma_old, action, zero, zero, adv, zero, weight, None), clip_ratio, False, dual_clip, 'k1',
        'ppoc'
    )
    return happo_policy_loss(loss.policy_loss, loss.entropy_loss), happo_info(info.approx_kl, info.clipfrac)
