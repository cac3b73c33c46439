"""``grpo_policy_error`` with the signature and namedtuples of ding/rl_utils/grpo.py -- csrc/vocab.cu.

With one of the three log-prob methods (ours or the reference's) the whole loss is ONE streaming launch over the three
(B, S, V) logit tensors that also writes d loss / d logit_new; any other ``log_prob_fn`` is called on the logits and the
kernel's token head runs on its (B, S) outputs, with autograd through the callable.  ``ppo.LAZY_INFO`` makes ``grpo_info``
carry 0-dim device tensors instead of python floats."""
from collections import namedtuple
from typing import Tuple

from . import _lm_policy
from .log_prob_utils import LogProbFunction, efficient_method

grpo_policy_data = namedtuple('grpo_policy_data', ['logit_new', 'logit_old', 'logit_ref', 'action', 'adv', 'weight'])
grpo_info = namedtuple('grpo_info', ['approx_kl', 'clipfrac'])


def grpo_policy_error(
        data: namedtuple,
        log_prob_fn: LogProbFunction = efficient_method,
        clip_ratio: float = 0.2,
        beta: float = 0.1
) -> Tuple[namedtuple, namedtuple]:
    """Group Relative Policy Optimization (https://arxiv.org/abs/2402.03300).  logit_new / logit_old / logit_ref
    (B, S, V) fp32 or bf16, action (B, S), adv (B), weight (B, S) or None.  Returns (loss, grpo_info(approx_kl,
    clipfrac)); loss = mean_b(sum_s(w * l) / sum_s(w)) with the per-token loss
    l = -min(r * adv, clamp(r, 1 - clip, 1 + clip) * adv) + beta * (exp(lp_ref - lp) - (lp_ref - lp) - 1)."""
    return _lm_policy.run((data.logit_new, data.logit_old, data.logit_ref), data.action, data.weight,
                          ('adv', data.adv), log_prob_fn, clip_ratio, beta, grpo_info)
