"""TEST INFRASTRUCTURE ONLY -- CPU restatement of the DQfD losses (ding/rl_utils/td.py:870-1090) and of R2D3's learner loop
over them (ding/policy/r2d3.py:322-388), with plain fp32 torch-CPU primitives in the reference's evaluation order, so that
on CPU it is bit-identical to the reference (``tests/test_dqfd.py::test_oracle_bit_exact_vs_reference``).  It builds on the
helpers of ``oracle/rl_oracle.py`` (the n-step return and the value transforms).  The product package never imports it.
Citations are ``file:line`` relative to ``ding/rl_utils/`` unless they name another file.
"""
import torch

from oracle.rl_oracle import nstep_return, value_inv_transform, value_transform


def dqfd_nstep_td_error(q, next_n_q, action, next_n_action, reward, done, done_one_step, weight, new_n_q_one_step,
                        next_n_action_one_step, is_expert, gamma: float, lambda_n_step_td: float,
                        lambda_supervised_loss: float, margin_function: float, lambda_one_step_td: float = 1.,
                        nstep: int = 1, cum_reward: bool = False, value_gamma=None, criterion=None, rescale: bool = False,
                        trans_fn=None, inv_trans_fn=None):
    """Both reference functions (``rescale`` selects the second; its transforms default to value_transform / _inv).
    Returns ``(loss, td_error_per_sample, (td_n.mean(), td_1.mean(), JE.mean()))``."""
    if criterion is None:
        criterion = torch.nn.MSELoss(reduction='none')
    trans_fn = trans_fn or value_transform
    inv_trans_fn = inv_trans_fn or value_inv_transform
    assert action.dim() == 1, action.shape  # td.py:933 / :1031
    if weight is None:
        weight = torch.ones_like(action)  # td.py:934-935 -- int64 ones
    rows = torch.arange(action.shape[0])
    q_sa = q[rows, action]  # td.py:938
    tq = next_n_q[rows, next_n_action]
    tq1 = new_n_q_one_step[rows, next_n_action_one_step]
    if rescale:  # td.py:1039, :1042
        tq = inv_trans_fn(tq)
        tq1 = inv_trans_fn(tq1)
    if cum_reward:  # td.py:943-947
        if value_gamma is None:
            tq = reward + (gamma ** nstep) * tq * (1 - done)
        else:
            tq = reward + value_gamma * tq * (1 - done)
    else:
        tq = nstep_return(reward, tq, done, gamma, nstep, value_gamma)  # td.py:949
    if rescale:
        tq = trans_fn(tq)  # td.py:1054
    td_n = criterion(q_sa, tq.detach())
    r1 = reward[0].unsqueeze(0)  # td.py:954: with cum_reward, sample 0's reward for every sample
    if cum_reward:  # td.py:956-960, value_gamma is None here
        tq1 = r1 + gamma * tq1 * (1 - done_one_step)
    else:
        tq1 = nstep_return(r1, tq1, done_one_step, gamma, 1, None)  # td.py:962-964
    if rescale:
        tq1 = trans_fn(tq1)  # td.py:1071
    td_1 = criterion(q_sa, tq1.detach())
    margin = margin_function * torch.ones_like(q)  # td.py:969-972
    margin.scatter_(1, action.unsqueeze(1), torch.zeros_like(q))
    je = is_expert * (torch.max(q + margin, dim=1)[0] - q_sa)
    loss = ((lambda_n_step_td * td_n + lambda_one_step_td * td_1 + lambda_supervised_loss * je) * weight).mean()
    per = lambda_n_step_td * td_n.abs() + lambda_one_step_td * td_1.abs() + lambda_supervised_loss * je.abs()
    return loss, per, (td_n.mean(), td_1.mean(), je.mean())  # td.py:974-983


def dqfd_nstep_td_error_sequence(q, next_n_q, action, next_n_action, reward, done, done_one_step, weight, new_n_q_one_step,
                                 next_n_action_one_step, is_expert, gamma: float, lambda_n_step_td: float,
                                 lambda_supervised_loss: float, margin_function: float, lambda_one_step_td: float = 1.,
                                 nstep: int = 1, value_gamma=None, rescale: bool = False, priority_mix: float = 0.9):
    """R2D3's learner loop (ding/policy/r2d3.py:322-388) with the parameters bound by name: q (T, B, N), reward
    (T, nstep, B), the rest (T, B).  Returns (loss, priority, td (T, B), (loss_n, loss_1, loss_sl))."""
    losses, errs, s_n, s_1, s_sl = [], [], [], [], []
    for t in range(q.shape[0]):  # r2d3.py:322
        l, e, s = dqfd_nstep_td_error(q[t], next_n_q[t], action[t], next_n_action[t], reward[t], done[t],
                                      done_one_step[t], None if weight is None else weight[t], new_n_q_one_step[t],
                                      next_n_action_one_step[t], is_expert[t], gamma, lambda_n_step_td,
                                      lambda_supervised_loss, margin_function, lambda_one_step_td, nstep, False,
                                      None if value_gamma is None else value_gamma[t], rescale=rescale)
        losses.append(l)
        errs.append(e)  # r2d3.py:353: no abs
        s_n.append(s[0])
        s_1.append(s[1])
        s_sl.append(s[2])
    div = len(losses) + 1e-8  # r2d3.py:379-383
    loss = sum(losses) / div
    stats = (sum(s_n) / div, sum(s_1) / div, sum(s_sl) / div)
    prio = priority_mix * torch.max(torch.stack(errs), dim=0)[0] + (1 - priority_mix) * (
        torch.sum(torch.stack(errs), dim=0) / (len(errs) + 1e-8))  # r2d3.py:386-388
    return loss, prio.detach(), torch.stack(errs), stats

