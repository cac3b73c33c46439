"""TEST INFRASTRUCTURE ONLY -- CPU restatement of the entropy-regularised TD losses of ding/rl_utils/td.py:
``m_q_1step_td_error`` (Munchausen DQN, :75-158), ``q_v_1step_td_error`` (the discrete SAC critic, :161-219) and
``q_nstep_sql_td_error`` (soft Q-learning, :1175-1245), in plain torch ops in the reference's evaluation order, so that in
fp32 on the CPU it is bit-identical to the reference (``tests/test_td_soft_dqfd_fp64.py::test_soft_td_oracle_*``), and in
float64 when the operands are float64 (every constant it builds takes the operands' or the default dtype).  The
signatures are the reference's, so callers written against the reference run on it unchanged.  The product package
never imports it.  Citations are ``file:line`` relative to ``ding/rl_utils/``.
"""
from collections import namedtuple

import torch
import torch.nn as nn

from oracle.rl_oracle import nstep_return

m_q_1step_td_data = namedtuple('m_q_1step_td_data', ['q', 'target_q', 'next_q', 'act', 'reward', 'done', 'weight'])
q_v_1step_td_data = namedtuple('q_v_1step_td_data', ['q', 'v', 'act', 'reward', 'done', 'weight'])
q_nstep_td_data = namedtuple('q_nstep_td_data', ['q', 'next_n_q', 'action', 'next_n_action', 'reward', 'done', 'weight'])


def _log_policy(x, tau):
    """tau * log softmax(x / tau) with the row max taken out first (td.py:129-132, :140-142); also returns x - max"""
    shifted = x - x.max(1)[0].unsqueeze(-1)
    return shifted, shifted - tau * torch.logsumexp(shifted / tau, 1).unsqueeze(-1)


def m_q_1step_td_error(data, gamma: float, tau: float, alpha: float, criterion=nn.MSELoss(reduction='none')):
    """-> (loss, td_error_per_sample (B,), action_gap, clipfrac (B, 1))"""
    q, target_q, next_q, act, reward, done, weight = data
    assert len(act.shape) == 1, act.shape  # td.py:121
    assert len(reward.shape) == 1, reward.shape  # td.py:122
    rows = torch.arange(act.shape[0])
    if weight is None:
        weight = torch.ones_like(reward)
    q_sa = q[rows, act]
    # Munchausen bonus: alpha * clamp(log pi(a | s), -1, 1) under the target network's current policy (td.py:129-137)
    _, log_pi = _log_policy(target_q, tau)
    log_pi_a = log_pi.gather(1, act.unsqueeze(-1))
    bonus = alpha * torch.clamp(log_pi_a, min=-1, max=1)
    # soft value of the next state: sum_j pi'_j * (q'_j - tau log pi'_j), masked by (1 - done) (td.py:140-145)
    shifted_next, tau_log_pi_next = _log_policy(next_q, tau)
    pi_next = torch.softmax(shifted_next / tau, dim=1)
    soft = (gamma * (pi_next * (next_q - tau_log_pi_next) * (1 - done.unsqueeze(-1))).sum(1)).unsqueeze(-1)
    target = reward.unsqueeze(-1) + bonus + soft  # td.py:147
    td = criterion(q_sa.unsqueeze(-1), target.detach()).squeeze(-1)
    with torch.no_grad():  # td.py:151-156
        top2 = target_q.topk(2, dim=1, largest=True, sorted=True)[0]
        action_gap = (top2[:, 0] - top2[:, 1]).mean()
        clipfrac = (log_pi_a.gt(1) | log_pi_a.lt(-1)).to(log_pi_a.dtype)
    return (td * weight).mean(), td, action_gap, clipfrac


def q_v_1step_td_error(data, gamma: float, criterion=nn.MSELoss(reduction='none')):
    """-> (loss, td_error_per_sample shaped like act); act (B,) or (B, A), reward / done (B,) (td.py:198-219)"""
    q, v, act, reward, done, weight = data
    assert len(reward.shape) == 1, reward.shape
    if act.dim() == 1:
        if weight is None:
            weight = torch.ones_like(reward)
        q_sa = q[torch.arange(act.shape[0]), act]
        target = gamma * (1 - done) * v + reward
    else:
        if weight is None:
            weight = torch.ones_like(act)
        B, A = act.shape
        q_sa = q.reshape(B * A, -1)[torch.arange(B * A), act.reshape(B * A)].reshape(B, A)
        target = gamma * (1 - done).unsqueeze(1) * v + reward.unsqueeze(1)
    td = criterion(q_sa, target.detach())
    return (td * weight).mean(), td


def q_nstep_sql_td_error(data, gamma: float, alpha: float, nstep: int = 1, cum_reward: bool = False, value_gamma=None,
                         criterion=nn.MSELoss(reduction='none')):
    """-> (loss, td_error_per_sample, record_target_v (B,)); the n-step return of V' = alpha * logsumexp(next_n_q / alpha)
    with +inf -> 20 and -inf -> -20 (td.py:1219-1245)"""
    q, next_n_q, action, next_n_action, reward, done, weight = data
    assert len(action.shape) == 1, action.shape  # td.py:1220
    if weight is None:
        weight = torch.ones_like(action)
    q_sa = q[torch.arange(action.shape[0]), action]
    v = alpha * torch.logsumexp(next_n_q / alpha, 1)
    v[v == float('inf')] = 20
    v[v == float('-inf')] = -20
    record_v = v.clone()
    if cum_reward:
        if value_gamma is None:
            v = reward + (gamma ** nstep) * v * (1 - done)
        else:
            v = reward + value_gamma * v * (1 - done)
    else:
        v = nstep_return(reward, v, done, gamma, nstep, value_gamma)
    td = criterion(q_sa, v.detach())
    return (td * weight).mean(), td, record_v
