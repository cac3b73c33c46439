"""``rloo_policy_error`` with the signature and namedtuples of ding/rl_utils/rloo.py -- csrc/vocab.cu.

The leave-one-out advantage is formed inside the kernel from reward (K, B'): row b = k * B' + j takes
r[k, j] - (sum_k' r[k', j] - r[k, j]) / (K - 1), the reference's ``adv.flatten()`` order.  Log-prob methods, custom
callables and ``ppo.LAZY_INFO`` as for ``grpo_policy_error``."""
from collections import namedtuple
from typing import Tuple

from . import _lm_policy
from .log_prob_utils import LogProbFunction, efficient_method

rloo_policy_data = namedtuple('rloo_policy_data', ['logit_new', 'logit_old', 'action', 'reward', 'weight'])
rloo_info = namedtuple('rloo_info', ['approx_kl', 'clipfrac'])


def rloo_policy_error(
        data: namedtuple,
        log_prob_fn: LogProbFunction = efficient_method,
        clip_ratio: float = 0.2,
) -> Tuple[namedtuple, namedtuple]:
    """REINFORCE Leave-One-Out (https://arxiv.org/abs/2402.14740).  logit_new / logit_old (B, S, V) fp32 or bf16, action
    (B, S), reward (K, B / K), weight (B, S) or None.  Returns (loss, rloo_info(approx_kl, clipfrac)) with the loss of
    ``grpo_policy_error`` without its KL term."""
    return _lm_policy.run((data.logit_new, data.logit_old), data.action, data.weight, ('reward', data.reward),
                          log_prob_fn, clip_ratio, 0.0, rloo_info)
