"""Quantile-regression n-step TD heads with the signatures of ding/rl_utils/td.py: ``qrdqn_nstep_td_error`` (:1098),
``iqn_nstep_td_error`` (:1253), ``fqf_nstep_td_error`` (:1359) -- one kernel (csrc/quantile.cu), the three tensor layouts are
handed over as strides, so no ``gather`` / ``permute`` / ``repeat`` copy is made.  FQF's fraction loss,
``fqf_calculate_fraction_loss`` (:1466), runs on its own kernel in the same file and reads its inputs through strides too."""
from collections import namedtuple
from typing import Optional

import torch

from .. import ops, torch_ops
from .td import _value_gamma_arg

qrdqn_nstep_td_data = namedtuple(
    'qrdqn_nstep_td_data', ['q', 'next_n_q', 'action', 'next_n_action', 'reward', 'done', 'tau', 'weight']
)
iqn_nstep_td_data = namedtuple(
    'iqn_nstep_td_data', ['q', 'next_n_q', 'action', 'next_n_action', 'reward', 'done', 'replay_quantiles', 'weight']
)
fqf_nstep_td_data = namedtuple(
    'fqf_nstep_td_data', ['q', 'next_n_q', 'action', 'next_n_action', 'reward', 'done', 'quantiles_hats', 'weight']
)


def _check(q, next_n_q, action, next_n_action, reward, done, nstep):
    # the reference's assertions (td.py:1133-1138), same messages
    assert len(action.shape) == 1, action.shape
    assert len(next_n_action.shape) == 1, next_n_action.shape
    assert len(done.shape) == 1, done.shape
    assert len(q.shape) == 3, q.shape
    assert len(next_n_q.shape) == 3, next_n_q.shape
    assert len(reward.shape) == 2, reward.shape
    assert reward.shape[0] == nstep


def _run(q, next_n_q, action, next_n_action, reward, done, tau, weight, gamma, nstep, value_gamma, form, kappa, axes):
    """``axes`` = positions of (sample, quantile, action) in q / next_n_q; ``tau`` already broadcast to (B, n_tau)."""
    dev = ops.compute_device(q, next_n_q)
    host_out = not q.is_cuda
    qd = ops.f32c(ops.to_device(q, dev), 'q')
    nq = ops.f32c(ops.to_device(next_n_q.detach(), dev), 'next_n_q')
    B, n_tau, N = (qd.shape[a] for a in axes)
    n_tau_p = nq.shape[axes[1]]
    if nq.shape[axes[0]] != B or nq.shape[axes[2]] != N or action.shape[0] != B or next_n_action.shape[0] != B \
            or done.shape[0] != B or reward.shape[1] != B:
        raise ValueError("quantile td: q %s / next_n_q %s / action %s / reward %s / done %s do not agree on (B, N)" %
                         (tuple(q.shape), tuple(next_n_q.shape), tuple(action.shape), tuple(reward.shape), tuple(done.shape)))
    act = ops.i64c(ops.to_device(action, dev), N)
    nact = ops.i64c(ops.to_device(next_n_action, dev), N, 'next_n_action')
    r = ops.f32c(ops.to_device(reward.detach(), dev), 'reward')
    d = ops.f32c(ops.to_device(done.detach(), dev), 'done')
    t = ops.to_device(tau.detach(), dev)
    if t.dtype != torch.float32:
        t = t.float()
    w = None
    if weight is not None:
        w = ops.f32c(ops.to_device(weight.detach(), dev), 'weight').reshape(-1)
        if w.numel() != B:
            raise ValueError("weight must have B=%d elements" % B)
    vg, vg_stride = _value_gamma_arg(value_gamma, B, dev)
    loss, td = torch_ops.quantile_td(qd, nq, act, nact, r, d, t, w, vg, vg_stride, B, N, n_tau, n_tau_p, nstep,
                                     float(gamma), form, float(kappa))
    return (loss.cpu(), td.cpu()) if host_out else (loss, td)


def qrdqn_nstep_td_error(
        data: namedtuple,
        gamma: float,
        nstep: int = 1,
        value_gamma: Optional[torch.Tensor] = None,
) -> torch.Tensor:
    """
    Drop-in for ding/rl_utils/td.py:1098-1166.  q, next_n_q (B, N, num) (the layout the body indexes, td.py:1145-1147);
    action, next_n_action, done (B,); reward (nstep, B); ``tau`` anything broadcastable to (B, num, 1) -- the (B, num, 1)
    quantile midpoints of the QRDQN head, or a python number as in the reference's own test (tests/test_td.py:252-260);
    weight None or (B,).  Returns (loss, td_error_per_sample (B,)), both attached to ``q``.
    """
    q, next_n_q, action, next_n_action, reward, done, tau, weight = data
    _check(q, next_n_q, action, next_n_action, reward, done, nstep)
    B, _, num = q.shape
    t = tau if isinstance(tau, torch.Tensor) else torch.as_tensor(tau, dtype=torch.float32)
    # tau meets u of shape (B, num, num') by broadcasting (td.py:1164); only its (b, i) plane can carry information
    t = torch.broadcast_to(t, (B, num, next_n_q.shape[2]))
    if t.stride(2) != 0 and t.shape[2] != 1:
        raise NotImplementedError("qrdqn_nstep_td_error: tau varies along the target-quantile axis")
    t = t[:, :, 0]
    return _run(q, next_n_q, action, next_n_action, reward, done, t, weight, gamma, nstep, value_gamma, 0, 1.0, (0, 2, 1))


def iqn_nstep_td_error(
        data: namedtuple,
        gamma: float,
        nstep: int = 1,
        kappa: float = 1.0,
        value_gamma: Optional[torch.Tensor] = None,
) -> torch.Tensor:
    """
    Drop-in for ding/rl_utils/td.py:1253-1346.  q (tau, B, N), next_n_q (tau', B, N), replay_quantiles (tau, B, 1) (any shape
    with tau * B elements, td.py:1335), action / next_n_action / done (B,), reward (nstep, B), weight None or (B,).
    Returns (loss, td_error_per_sample (B,)), both attached to ``q``.
    """
    q, next_n_q, action, next_n_action, reward, done, replay_quantiles, weight = data
    _check(q, next_n_q, action, next_n_action, reward, done, nstep)
    tau, B = q.shape[0], done.shape[0]
    t = replay_quantiles.reshape(tau, B).t()  # (B, tau) view: strides only
    return _run(q, next_n_q, action, next_n_action, reward, done, t, weight, gamma, nstep, value_gamma, 1, kappa, (1, 0, 2))


def fqf_nstep_td_error(
        data: namedtuple,
        gamma: float,
        nstep: int = 1,
        kappa: float = 1.0,
        value_gamma: Optional[torch.Tensor] = None,
) -> torch.Tensor:
    """
    Drop-in for ding/rl_utils/td.py:1359-1436.  q (B, tau, N), next_n_q (B, tau', N), quantiles_hats (B, tau), action /
    next_n_action / done (B,), reward (nstep, B), weight None or (B,).  Returns (loss, td_error_per_sample (B,)), both
    attached to ``q``.
    """
    q, next_n_q, action, next_n_action, reward, done, quantiles_hats, weight = data
    _check(q, next_n_q, action, next_n_action, reward, done, nstep)
    B, tau = q.shape[0], q.shape[1]
    t = quantiles_hats.expand(B, tau)
    return _run(q, next_n_q, action, next_n_action, reward, done, t, weight, gamma, nstep, value_gamma, 2, kappa, (0, 1, 2))


def _f32(t, name):
    # fp32 as it is, views included: the kernel reads through strides
    return t if t.dtype == torch.float32 else ops.f32c(t, name)


def _gather_check(q_s, actions):
    # evaluate_quantile_at_action (td.py:1452-1463): its assertion, and the shapes its gather accepts
    assert q_s.shape[0] == actions.shape[0]
    if q_s.dim() != 3 or actions.dim() != 1:
        raise RuntimeError("fqf_calculate_fraction_loss: gather needs a (B, n, A) tensor and (B,) actions, got %s and %s" %
                           (tuple(q_s.shape), tuple(actions.shape)))


def fqf_calculate_fraction_loss(q_tau_i, q_value, quantiles, actions):
    """
    Drop-in for ding/rl_utils/td.py:1466-1513.  q_tau_i (B, N-1, A), q_value (B, N, A) (must require grad; neither gets a
    gradient), quantiles (B, N+1), actions (B,).  Returns the fraction loss, a 0-dim tensor attached to ``quantiles`` only
    (no grad_fn when quantiles does not require grad).
    """
    assert q_value.requires_grad
    batch_size, num_quantiles = q_value.shape[0], q_value.shape[1]
    _gather_check(q_tau_i, actions)
    assert (q_tau_i.shape[0], q_tau_i.shape[1]) == (batch_size, num_quantiles - 1)  # td.py:1487
    _gather_check(q_value, actions)
    assert quantiles[:, 1:-1].shape == (batch_size, num_quantiles - 1)  # td.py:1507
    dev = ops.compute_device(q_tau_i, q_value, quantiles, actions)
    host_out = not quantiles.is_cuda
    qt = _f32(ops.to_device(q_tau_i.detach(), dev), 'q_tau_i')
    qv = _f32(ops.to_device(q_value.detach(), dev), 'q_value')
    qn = _f32(ops.to_device(quantiles, dev), 'quantiles')
    act = ops.i64c(ops.to_device(actions, dev), min(qt.shape[2], qv.shape[2]), 'actions')
    loss = torch_ops.fqf_fraction(qt, qv, qn, act, batch_size, num_quantiles)
    return loss.cpu() if host_out else loss
