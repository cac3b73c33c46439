"""n-step TD operators with the signatures of ding/rl_utils/td.py -- kernels in csrc/td.cu.

  q_nstep_td_error (td.py:649-719), q_nstep_td_error_with_rescale (:810-867), dist_nstep_td_error (:413-523),
  td_lambda_error (:1539-1571), generalized_lambda_returns (:1574-1605),
  and the 1-step / state-value siblings that reuse the q-n-step kernels (SURVEY section 8f rank 2):
  q_1step_td_error (:26-72), v_1step_td_error (:529-573), v_nstep_td_error (:579-617);
  dqfd_nstep_td_error (:870-983) / dqfd_nstep_td_error_with_rescale (:986-1090) on their own kernel (dqfd_fwd / dqfd_bwd);
  m_q_1step_td_error (:75-158), q_nstep_sql_td_error (:1175-1245) and q_v_1step_td_error (:161-219) on one forward kernel
  (soft_td_fwd) and the q-n-step backward.
"""
from collections import namedtuple
from typing import Callable, Optional, Union

import torch
import torch.nn as nn

from .. import ops, torch_ops
from .value_rescale import value_inv_transform, value_transform

q_nstep_td_data = namedtuple(
    'q_nstep_td_data', ['q', 'next_n_q', 'action', 'next_n_action', 'reward', 'done', 'weight']
)
# the reference's typename string is 'dist_1step_td_data' (td.py:386-388); kept for pickling / repr compatibility
dist_nstep_td_data = namedtuple(
    'dist_1step_td_data', ['dist', 'next_n_dist', 'act', 'next_n_act', 'reward', 'done', 'weight']
)
dist_1step_td_data = namedtuple(
    'dist_1step_td_data', ['dist', 'next_dist', 'act', 'next_act', 'reward', 'done', 'weight']
)
td_lambda_data = namedtuple('td_lambda_data', ['value', 'reward', 'weight'])
q_1step_td_data = namedtuple('q_1step_td_data', ['q', 'next_q', 'act', 'next_act', 'reward', 'done', 'weight'])
v_1step_td_data = namedtuple('v_1step_td_data', ['v', 'next_v', 'reward', 'done', 'weight'])
v_nstep_td_data = namedtuple('v_nstep_td_data', ['v', 'next_n_v', 'reward', 'done', 'weight', 'value_gamma'])

# The reference asserts ``dist[b, act] > 0`` on the host every call (td.py:513).  True keeps that behaviour (one
# 4-byte D2H read per call); False skips the read -- a non-positive entry then shows up as nan/inf in the loss.
CHECK_DIST_POSITIVE = True

_SUPPORT_CACHE = {}


def _data(args, kwargs):
    return args[0] if len(args) > 0 else kwargs['data']


def shape_fn_qntd(args, kwargs):
    """[T, B, N] cache key (td.py:632-645)."""
    d = _data(args, kwargs)
    return [d.reward.shape[0]] + list(d.q.shape)


def shape_fn_qntd_rescale(args, kwargs):
    """[T, B, N] cache key (td.py:791-804)."""
    d = _data(args, kwargs)
    return [d.reward.shape[0]] + list(d.q.shape)


def shape_fn_dntd(args, kwargs):
    """[T, B, N, n_atom] cache key (td.py:391-404)."""
    d = _data(args, kwargs)
    return [d.reward.shape[0]] + list(d.dist.shape)


def shape_fn_td_lambda(args, kwargs):
    """(T, B) cache key; the keyword form returns only T, exactly like the reference (td.py:1519-1529)."""
    if len(args) <= 0:
        return kwargs['data'].reward.shape[0]
    return args[0].reward.shape


def _criterion_code(criterion):
    """Map a torch criterion module to the fused kernel's enum; None when it has to run as a torch module."""
    if getattr(criterion, 'reduction', None) != 'none':
        return None
    if type(criterion) is nn.MSELoss:
        return 0, 0.0
    if type(criterion) is nn.L1Loss:
        return 1, 0.0
    if type(criterion) is nn.SmoothL1Loss:
        beta = float(criterion.beta)
        return (2, beta) if beta > 0 else (1, 0.0)
    if type(criterion) is nn.HuberLoss:
        return 3, float(criterion.delta)
    return None


def _value_gamma_arg(value_gamma, B, dev):
    """-> (tensor or None, stride): None | python scalar | 0-dim / 1-element tensor (stride 0) | (B,) tensor (stride 1)."""
    if value_gamma is None:
        return None, 0
    if not isinstance(value_gamma, torch.Tensor):
        return ops.const_scalar(value_gamma, dev), 0
    vg = ops.f32c(ops.to_device(value_gamma.detach(), dev), 'value_gamma')
    if vg.numel() == 1:
        return vg.reshape(1), 0
    if vg.numel() != B:
        raise ValueError("value_gamma must have 1 or B=%d elements, got %s" % (B, tuple(value_gamma.shape)))
    return vg.reshape(B), 1


def _value_gamma_op_arg(value_gamma, B, dev):
    """``_value_gamma_arg`` for the custom ops (rl_utils' traced path): a python scalar stays a float, which the op reads
    from the cached device constant when it runs, so that tracing allocates nothing"""
    if value_gamma is not None and not isinstance(value_gamma, torch.Tensor):
        return float(value_gamma), 0
    return _value_gamma_arg(value_gamma, B, dev)


def _gamma_arg(gamma, B, dev, cum_reward):
    """python float -> (gamma, None); the NGU list of B 0-dim tensors (td.py:275-282) -> (0.0, (B,) device tensor)."""
    if isinstance(gamma, float):
        return gamma, None
    if isinstance(gamma, list):
        if cum_reward:
            raise TypeError("cum_reward with a list gamma is not defined by the reference (td.py:711-715)")
        gamma_ps = ops.f32c(torch.stack([torch.as_tensor(g) for g in gamma], dim=0).to(dev), 'gamma').reshape(-1)
        if gamma_ps.numel() != B:
            raise ValueError("list gamma must have B=%d entries" % B)
        return 0.0, gamma_ps
    raise TypeError("The type of gamma should be float or list")


def _qntd_rows(q, next_n_q, action, next_n_action, reward, done, weight, value_gamma, gamma, nstep, cum_reward,
               criterion, rescale, trans_fn=None, inv_trans_fn=None, group_mean=False):
    """The canonical row form every public signature below is brought to: q, next_n_q (S, G, N); action, next_n_action
    (S, G); reward (nstep, S) -- (S,) with cum_reward; done, weight (S,); value_gamma None | scalar | 1-element | (S,).
    Returns (loss, td) with td (S, G), or (S,) = mean over G with ``group_mean``; both carry gradient to ``q``."""
    dev = ops.compute_device(q, next_n_q)
    S, G, N = q.shape
    gamma_f, gamma_ps = _gamma_arg(gamma, S, dev, cum_reward)
    qd = ops.f32c(ops.to_device(q, dev), 'q')
    nq = ops.f32c(ops.to_device(next_n_q.detach(), dev), 'next_n_q')
    act = ops.i64c(ops.to_device(action, dev), q.shape[-1])
    nact = ops.i64c(ops.to_device(next_n_action, dev), q.shape[-1], 'next_n_action')
    r = ops.f32c(ops.to_device(reward.detach(), dev), 'reward')
    d = ops.f32c(ops.to_device(done.detach(), dev), 'done')
    if (nq.shape != qd.shape or act.numel() != S * G or nact.numel() != S * G or
            r.numel() != (S if cum_reward else nstep * S) or d.numel() != S):
        raise ValueError("q %s / next_n_q %s / action %s / next_n_action %s / reward %s / done %s do not match "
                         "S=%d, G=%d, nstep=%d" % (tuple(q.shape), tuple(next_n_q.shape), tuple(action.shape),
                                                   tuple(next_n_action.shape), tuple(reward.shape), tuple(done.shape),
                                                   S, G, nstep))
    w = None
    if weight is not None:
        w = ops.f32c(ops.to_device(weight.detach(), dev), 'weight')
        if w.numel() != S:
            w = w.expand(S).contiguous()
    vg, vg_stride = (_value_gamma_op_arg if torch.compiler.is_compiling() else _value_gamma_arg)(value_gamma, S, dev)
    custom_trans = rescale and (trans_fn is not value_transform or inv_trans_fn is not value_inv_transform)
    code = _criterion_code(criterion)
    gm = 1 if group_mean else 0

    def kernel(q_, nq_, act_, nact_, n_, resc, crit, param):
        if torch.compiler.is_compiling():
            return torch_ops.qntd(q_, nq_, act_, nact_, r, d, w, vg, vg_stride, gamma_ps, S, G, n_, int(nstep),
                                  float(gamma_f), 1 if cum_reward else 0, resc, 1e-2, crit, param, gm) + (None, )
        return ops.QNStepTDFunction.apply(q_, nq_, act_, nact_, r, d, w, vg, vg_stride, gamma_ps, S, G, n_, int(nstep),
                                          float(gamma_f), 1 if cum_reward else 0, resc, 1e-2, crit, param, gm, 0, 0.0,
                                          False)

    if custom_trans or code is None:
        # user-supplied transforms / criterion are torch callables: the kernel produces the detached n-step target (of the
        # inverse-transformed next value), the callables run on the device around it
        wb = w.reshape(S, 1) if w is not None else 1.0
        if custom_trans:
            tq = inv_trans_fn(nq.gather(-1, nact.reshape(S, G, 1))).reshape(S, G, 1).contiguous()
            zero = torch.zeros(S, G, dtype=torch.int64, device=dev)
            _, _, target, _ = kernel(qd.detach().gather(-1, act.reshape(S, G, 1)).contiguous(), tq, zero, zero, 1, 0, 0,
                                     0.0)
            target = trans_fn(target.reshape(S, G)).detach()
        else:
            _, _, target, _ = kernel(qd.detach(), nq, act, nact, N, 1 if rescale else 0, 0, 0.0)
            target = target.reshape(S, G)
        per = criterion(qd.gather(-1, act.reshape(S, G, 1)).squeeze(-1), target)
        loss = (per * wb).mean()
        if group_mean:
            per = per.mean(-1)
        return loss, per
    loss, per, _, _ = kernel(qd, nq, act, nact, N, 1 if rescale else 0, code[0], code[1])
    return loss, (per if group_mean else per.reshape(S, G))


def _qntd(data, gamma, nstep, cum_reward, value_gamma, criterion, rescale, trans_fn=None, inv_trans_fn=None):
    """q_nstep_td_error / _with_rescale: the common (B, N) / (B,) call goes straight to the row form; every other shape the
    reference accepts (td.py:692-719) is first broadcast exactly as the reference's tensor expressions broadcast it."""
    q, next_n_q, action, next_n_action, reward, done, weight = data
    host_out = not q.is_cuda
    if not isinstance(gamma, (float, list)):
        raise TypeError("The type of gamma should be float or list")
    if not cum_reward:
        assert reward.shape[0] == nstep  # td.py:257
    B = q.shape[0]
    plain = (q.dim() == 2 and action.dim() == 1 and next_n_action.dim() == 1 and done.dim() == 1 and
             tuple(reward.shape) == ((B, ) if cum_reward else (nstep, B)) and
             (weight is None or weight.numel() in (1, B)))
    if plain:
        N = q.shape[1]
        loss, per = _qntd_rows(q.reshape(B, 1, N), next_n_q.reshape(B, 1, N), action.reshape(B, 1),
                               next_n_action.reshape(B, 1), reward, done, weight, value_gamma, gamma, nstep, cum_reward,
                               criterion, rescale, trans_fn, inv_trans_fn)
        per = per.reshape(B)
    else:
        loss, per = _qntd_general(q, next_n_q, action, next_n_action, reward, done, weight, value_gamma, gamma, nstep,
                                  cum_reward, criterion, rescale, trans_fn, inv_trans_fn)
    if host_out:
        loss, per = loss.cpu(), per.cpu()
    return loss, per


def _qntd_general(q, next_n_q, action, next_n_action, reward, done, weight, value_gamma, gamma, nstep, cum_reward,
                  criterion, rescale, trans_fn, inv_trans_fn):
    """Shapes beyond (B, N) / (B,): the reference evaluates q_nstep_td_error with broadcasting tensor expressions, so e.g.
    ``cum_reward=True`` with an (nstep, B) reward (its own test, tests/test_td.py:29-35) yields an (nstep, B) error, and the
    multi-agent branch (action (B, A, 1) against q (B, A, N), td.py:700-705) a (B, A) one.  Here the shape algebra of
    td.py:692-719 / :230-286 is replayed on the host (shapes only -- an incompatible combination raises the same
    broadcasting ``RuntimeError`` the reference raises), every operand is expanded to the resulting error shape and the
    rows go through the same kernel.  Expansion is a view + copy; the gradient of an expanded ``q`` is reduced by autograd."""
    bs = torch.broadcast_shapes
    weight_given = weight is not None
    w_shape = tuple(weight.shape) if weight_given else tuple(reward.shape)  # td.py:693 ones_like(reward)
    r_shape, d_shape = tuple(reward.shape), tuple(done.shape)
    vg_t = value_gamma if isinstance(value_gamma, torch.Tensor) else None
    vg_shape = tuple(vg_t.shape) if vg_t is not None else None
    act = action
    if action.dim() == 1 or action.dim() < q.dim():
        act = action.unsqueeze(-1)
    elif action.dim() > 1:  # the reference's multi-agent branch
        r_shape, w_shape, d_shape = r_shape + (1, ), w_shape + (1, ), d_shape + (1, )
        if vg_shape is not None:
            vg_shape = vg_shape + (1, )
    if act.dim() != q.dim() or tuple(act.shape[:-1]) != tuple(q.shape[:-1]) or act.shape[-1] != 1:
        raise RuntimeError("gather: action %s does not index q %s" % (tuple(action.shape), tuple(q.shape)))
    if tuple(next_n_action.shape) != tuple(next_n_q.shape[:-1]):
        raise RuntimeError("gather: next_n_action %s does not index next_n_q %s" %
                           (tuple(next_n_action.shape), tuple(next_n_q.shape)))
    qsa_shape, tq_shape = tuple(q.shape[:-1]), tuple(next_n_q.shape[:-1])

    def trail(shape, like):  # view_similar, td.py:222-224
        return tuple(shape) + (1, ) * (len(like) - len(shape))

    # each operand's shape as it enters the final (broadcasting) expression
    if cum_reward:
        rew_term = r_shape
        if vg_shape is None:
            val_term = bs(tq_shape, d_shape)
            vg_b, d_b = None, d_shape
        else:
            val_term = bs(vg_shape, tq_shape, d_shape)
            vg_b, d_b = vg_shape, d_shape
    else:
        rew_term = r_shape[1:]  # reward.mul(reward_factor).sum(0)
        if isinstance(gamma, list):
            g_b = trail((d_shape[0], ), r_shape[1:])  # reward_factor[nstep] of view_similar(reward_factor, reward)
            val_term = bs(g_b, tq_shape, d_shape)
            vg_b, d_b = None, d_shape
        elif value_gamma is None:
            val_term = bs(tq_shape, d_shape)
            vg_b, d_b = None, d_shape
        else:
            vg_b = trail(vg_shape if vg_shape is not None else tq_shape, tq_shape)  # np.isscalar -> full_like(next_value)
            d_b = trail(d_shape, tq_shape)
            val_term = bs(vg_b, tq_shape, d_b)
    td_shape = bs(qsa_shape, bs(rew_term, val_term))
    if bs(td_shape, w_shape) != td_shape:
        if weight_given:
            raise ValueError("weight %s does not broadcast to the td error shape %s" % (w_shape, tuple(td_shape)))
        # ones_like(reward) against a smaller error: the mean of the broadcast product is the plain mean
    S = 1
    for n_ in td_shape:
        S *= n_
    N = q.shape[-1]
    dev = ops.compute_device(q, next_n_q)

    def rows(x, shape, lead=()):  # expand `x` (viewed as `shape`) to lead + td_shape and flatten the td dims
        x = ops.to_device(x, dev)
        return x.reshape(tuple(lead) + tuple(shape)).expand(tuple(lead) + tuple(td_shape)).reshape(tuple(lead) + (S, ))

    q_rows = ops.to_device(q, dev).reshape(qsa_shape + (N, )).expand(tuple(td_shape) + (N, )).reshape(S, 1, N)
    nq_rows = ops.to_device(next_n_q, dev).expand(tuple(td_shape) + (N, )).reshape(S, 1, N)
    a_rows = rows(act.squeeze(-1), qsa_shape).reshape(S, 1)
    na_rows = rows(next_n_action, tq_shape).reshape(S, 1)
    r_rows = rows(reward, r_shape) if cum_reward else rows(reward, r_shape[1:], lead=(nstep, ))
    d_rows = rows(done.float(), d_b)
    w_rows = rows(weight, w_shape) if weight_given else None
    gam = gamma
    if isinstance(gamma, list):
        gam = list(rows(torch.stack([torch.as_tensor(g) for g in gamma], 0).float(), g_b))
    vg_rows = value_gamma
    if vg_t is not None and vg_t.numel() > 1:
        vg_rows = rows(vg_t, vg_b)
    loss, per = _qntd_rows(q_rows, nq_rows, a_rows, na_rows, r_rows, d_rows, w_rows, vg_rows, gam, nstep, cum_reward,
                           criterion, rescale, trans_fn, inv_trans_fn)
    return loss, per.reshape(tuple(td_shape))


def q_nstep_td_error(
        data: namedtuple,
        gamma: Union[float, list],
        nstep: int = 1,
        cum_reward: bool = False,
        value_gamma: Optional[torch.Tensor] = None,
        criterion: torch.nn.modules = nn.MSELoss(reduction='none'),
) -> torch.Tensor:
    """
    Multi-step TD error for Q-learning, drop-in for ding/rl_utils/td.py:649-719 (n-step return :230-286).

    Shapes: q, next_n_q (B, N); action, next_n_action (B,) int64; reward (nstep, B) -- (B,) with ``cum_reward``;
    done (B,) (a float multiplier, as the reference's tests pass it); weight (B,) or None; value_gamma None, scalar
    or (B,); gamma float, or the NGU list of B 0-dim tensors.  Every other shape combination the reference's
    broadcasting expressions accept is accepted too and gives the reference's result shape: ``cum_reward=True`` with an
    (nstep, B) reward (tests/test_td.py:29-35) -> (nstep, B) errors; the multi-agent branch q (B, A, N) with action
    (B, A, 1) (td.py:700-705) -> (B, A) errors; incompatible shapes raise the reference's broadcasting ``RuntimeError``.
    Returns ``(loss, td_error_per_sample)``, both differentiable w.r.t. ``q`` as in the reference (td.py:718-719).
    """
    return _qntd(data, gamma, nstep, cum_reward, value_gamma, criterion, rescale=False)


def q_nstep_td_error_with_rescale(
    data: namedtuple,
    gamma: Union[float, list],
    nstep: int = 1,
    value_gamma: Optional[torch.Tensor] = None,
    criterion: torch.nn.modules = nn.MSELoss(reduction='none'),
    trans_fn: Callable = value_transform,
    inv_trans_fn: Callable = value_inv_transform,
) -> torch.Tensor:
    """
    Multi-step TD error with value rescaling h / h^-1, drop-in for ding/rl_utils/td.py:810-867.
    With the default transforms everything (h^-1, n-step return, h, criterion) runs in one kernel.
    """
    assert len(data.action.shape) == 1, data.action.shape  # td.py:854
    return _qntd(data, gamma, nstep, False, value_gamma, criterion, True, trans_fn, inv_trans_fn)


def q_1step_td_error(
        data: namedtuple,
        gamma: float,
        criterion: torch.nn.modules = nn.MSELoss(reduction='none'),
) -> torch.Tensor:
    """
    1-step TD error for Q-learning, drop-in for ding/rl_utils/td.py:26-72: ``target = gamma*(1-done)*next_q[next_act] +
    reward`` -- the n = 1 case of ``q_nstep_td_error`` (the reference pins that identity, tests/test_td.py:113-126), on the
    same kernel.  q, next_q (B, N); act, next_act (B,) int64; reward, done (B,); weight (B,) or None.  Returns the loss only.
    """
    q, next_q, act, next_act, reward, done, weight = data
    assert len(act.shape) == 1, act.shape        # td.py:64
    assert len(reward.shape) == 1, reward.shape  # td.py:65
    loss, _ = _qntd(q_nstep_td_data(q, next_q, act, next_act, reward.unsqueeze(0), done, weight), gamma, 1, False, None,
                    criterion, False)
    return loss


def bdq_nstep_td_error(
        data: namedtuple,
        gamma: Union[float, list],
        nstep: int = 1,
        cum_reward: bool = False,
        value_gamma: Optional[torch.Tensor] = None,
        criterion: torch.nn.modules = nn.MSELoss(reduction='none'),
) -> torch.Tensor:
    """
    Multi-step TD error of the branching dueling Q-network (BDQ), drop-in for ding/rl_utils/td.py:722-789:
    q, next_n_q (B, D, N) -- D action branches of N bins; action, next_n_action (B, D); reward (nstep, B) -- (B,) with
    ``cum_reward``; done (B,); weight (B,) or None.  Every branch shares the sample's n-step reward; the per-sample error is
    the mean over the branches (td.py:788).  Returns ``(loss, td_error_per_sample (B,))``.  One launch on the q-n-step kernel
    (G = D rows per sample).
    """
    q, next_n_q, action, next_n_action, reward, done, weight = data
    host_out = not q.is_cuda
    if not isinstance(gamma, (float, list)):
        raise TypeError("The type of gamma should be float or list")
    if not cum_reward:
        assert reward.shape[0] == nstep  # td.py:257
    B = q.shape[0]
    if q.dim() != 3 or action.dim() != 2 or tuple(action.shape) != tuple(q.shape[:2]):
        raise RuntimeError("bdq_nstep_td_error: q %s / action %s must be (B, D, N) / (B, D)" %
                           (tuple(q.shape), tuple(action.shape)))
    if tuple(reward.shape) == ((B, ) if cum_reward else (nstep, B)):
        loss, per = _qntd_rows(q, next_n_q, action, next_n_action, reward, done, weight, value_gamma, gamma, nstep,
                               cum_reward, criterion, False, group_mean=True)
    elif cum_reward and reward.dim() == 2 and reward.shape[1] == B:
        # (K, B) reward with cum_reward (tests/test_td.py:58-66): the reference broadcasts to a (K, B, D) error and averages
        # the branches -> (K, B); the K reward rows are K independent sample sets of the same q
        K, D, N = reward.shape[0], q.shape[1], q.shape[2]
        dev = ops.compute_device(q, next_n_q)

        def rep(x):
            x = ops.to_device(x, dev)
            return x.unsqueeze(0).expand((K, ) + tuple(x.shape)).reshape((K * B, ) + tuple(x.shape[1:]))

        vg = value_gamma
        if isinstance(vg, torch.Tensor) and vg.numel() > 1:
            vg = rep(vg)
        w = weight
        if w is not None:
            if tuple(w.shape) != (B, ):
                raise ValueError("weight %s does not broadcast to the td error shape %s" % (tuple(w.shape), (K, B)))
            w = rep(w)
        loss, per = _qntd_rows(rep(q), rep(next_n_q), rep(action), rep(next_n_action), ops.to_device(reward, dev).reshape(-1),
                               rep(done.float()), w, vg, gamma, nstep, True, criterion, False, group_mean=True)
        per = per.reshape(K, B)
    else:
        raise RuntimeError("bdq_nstep_td_error: reward %s does not match B=%d, nstep=%d" % (tuple(reward.shape), B, nstep))
    if host_out:
        loss, per = loss.cpu(), per.cpu()
    return loss, per


q_nstep_td_seq_data = namedtuple(
    'q_nstep_td_seq_data', ['q', 'next_n_q', 'action', 'next_n_action', 'reward', 'done', 'weight']
)


def q_nstep_td_error_sequence(
        data: namedtuple,
        gamma: Union[float, list],
        nstep: int = 1,
        value_gamma: Optional[torch.Tensor] = None,
        rescale: bool = False,
        priority_mix: float = 0.9,
        criterion: torch.nn.modules = nn.MSELoss(reduction='none'),
):
    """
    The per-time-step loop of the recurrent Q-learners in ONE launch.  Not a reference function: it is exactly what
    ``R2D2Policy._forward_learn`` / NGU / R2D3 compute around the operator (ding/policy/r2d2.py:347-369, ngu.py:330-360)::

        for t in range(T):
            l, e = q_nstep_td_error[_with_rescale](q_nstep_td_data(q[t], next_n_q[t], action[t], next_n_action[t],
                                                   reward[t], done[t], weight[t]), gamma, nstep, value_gamma=value_gamma[t])
            loss.append(l); td_error.append(e.abs())
        loss = sum(loss) / (len(loss) + 1e-8)
        priority = mix * max_t(td_error) + (1 - mix) * sum_t(td_error) / (len(td_error) + 1e-8)

    Shapes: q, next_n_q (T, B, N); action, next_n_action (T, B); reward (T, nstep, B) (the policy's permuted layout,
    r2d2.py:343); done, weight (T, B) (weight may be None); value_gamma (T, B) or None; gamma float or the NGU list of B
    0-dim tensors.  Returns ``(loss, priority (B,), td_error (T, B))``: loss and td_error carry gradient to ``q``; the
    priority (the replay priority) is detached.
    """
    q, next_n_q, action, next_n_action, reward, done, weight = data
    host_out = not q.is_cuda
    if q.dim() != 3 or action.dim() != 2 or reward.dim() != 3:
        raise ValueError("q_nstep_td_error_sequence: expected q (T, B, N), action (T, B), reward (T, nstep, B); got %s / %s "
                         "/ %s" % (tuple(q.shape), tuple(action.shape), tuple(reward.shape)))
    T, B, N = q.shape
    assert reward.shape[1] == nstep  # td.py:257 for every step
    dev = ops.compute_device(q, next_n_q)
    gamma_f, gamma_ps = _gamma_arg(gamma, B, dev, False)
    code = _criterion_code(criterion)
    if code is None:
        raise NotImplementedError("q_nstep_td_error_sequence: criterion must be MSELoss / L1Loss / SmoothL1Loss / HuberLoss "
                                  "with reduction='none'")
    qd = ops.f32c(ops.to_device(q, dev), 'q')
    nq = ops.f32c(ops.to_device(next_n_q.detach(), dev), 'next_n_q')
    act = ops.i64c(ops.to_device(action, dev), q.shape[-1])
    nact = ops.i64c(ops.to_device(next_n_action, dev), q.shape[-1], 'next_n_action')
    r = ops.f32c(ops.to_device(reward.detach(), dev), 'reward')
    d = ops.f32c(ops.to_device(done.detach(), dev), 'done')
    S = T * B
    if (nq.shape != qd.shape or tuple(act.shape) != (T, B) or tuple(nact.shape) != (T, B) or
            tuple(r.shape) != (T, nstep, B) or d.numel() != S):
        raise ValueError("q_nstep_td_error_sequence: operand shapes do not match T=%d, B=%d, nstep=%d" % (T, B, nstep))
    w = None
    if weight is not None:
        w = ops.f32c(ops.to_device(weight.detach(), dev), 'weight')
        if w.numel() != S:
            w = w.expand(T, B).contiguous()
    if torch.compiler.is_compiling():
        vg, vg_stride = _value_gamma_op_arg(value_gamma, S, dev)
        loss, per, prio = torch_ops.qntd_seq(qd, nq, act, nact, r, d, w, vg, vg_stride, gamma_ps, S, N, int(nstep),
                                             float(gamma_f), 1 if rescale else 0, code[0], code[1], T, float(priority_mix))
    else:
        vg, vg_stride = _value_gamma_arg(value_gamma, S, dev)
        loss, per, _, prio = ops.QNStepTDFunction.apply(
            qd, nq, act, nact, r, d, w, vg, vg_stride, gamma_ps, S, 1, N, int(nstep), float(gamma_f), 0,
            1 if rescale else 0, 1e-2, code[0], code[1], 0, T, float(priority_mix), True
        )
    per = per.reshape(T, B)
    if host_out:
        loss, prio, per = loss.cpu(), prio.cpu(), per.cpu()
    return loss, prio, per


dqfd_nstep_td_data = namedtuple(
    'dqfd_nstep_td_data', [
        'q', 'next_n_q', 'action', 'next_n_action', 'reward', 'done', 'done_one_step', 'weight', 'new_n_q_one_step',
        'next_n_action_one_step', 'is_expert'
    ]
)
dqfd_nstep_td_seq_data = namedtuple('dqfd_nstep_td_seq_data', dqfd_nstep_td_data._fields)


def _dqfd_operands(data, S, dev, rows):
    """Stage the operands of dqfd_nstep_td_data on ``dev``: q keeps its gradient, the rest are detached; ``rows`` is the
    (T, B) / (B,) shape of the per-sample operands.  is_expert (float, int or bool tensor, or a python scalar) is
    widened to float, as the reference's ``is_expert * (...)`` promotes it."""
    q, next_n_q, action, next_n_action, reward, done, done_one_step, weight, next_q1, next_action1, is_expert = data
    N = q.shape[-1]
    qd = ops.f32c(ops.to_device(q, dev), 'q')
    nq = ops.f32c(ops.to_device(next_n_q.detach(), dev), 'next_n_q')
    nq1 = ops.f32c(ops.to_device(next_q1.detach(), dev), 'new_n_q_one_step')
    act = ops.i64c(ops.to_device(action, dev), N)
    nact = ops.i64c(ops.to_device(next_n_action, dev), N, 'next_n_action')
    nact1 = ops.i64c(ops.to_device(next_action1, dev), N, 'next_n_action_one_step')
    r = ops.f32c(ops.to_device(reward.detach(), dev), 'reward')
    d = ops.f32c(ops.to_device(done.detach(), dev), 'done')
    d1 = ops.f32c(ops.to_device(done_one_step.detach(), dev), 'done_one_step')
    if not isinstance(is_expert, torch.Tensor):
        # traced: a float, which the custom op reads from the cached device constant when it runs
        ie = float(is_expert) if torch.compiler.is_compiling() else ops.const_scalar(is_expert, dev).expand(S).contiguous()
    else:
        ie = ops.f32c(ops.to_device(is_expert.detach(), dev), 'is_expert')
    if isinstance(ie, torch.Tensor) and ie.numel() == 1:
        ie = ie.reshape(1).expand(S).contiguous()
    ie_shape = tuple(ie.shape) if isinstance(ie, torch.Tensor) else (S, )
    w = None
    if weight is not None:
        w = ops.f32c(ops.to_device(weight.detach(), dev), 'weight')
        if w.numel() == 1:
            w = w.reshape(1).expand(S).contiguous()
    shape = tuple(qd.shape[:-1])
    if (shape != tuple(rows) or nq.shape != qd.shape or nq1.shape != qd.shape or tuple(act.shape) != shape or
            tuple(nact.shape) != shape or tuple(nact1.shape) != shape or d.numel() != S or d1.numel() != S or
            (isinstance(ie, torch.Tensor) and ie.numel() != S) or (w is not None and w.numel() != S)):
        raise ValueError("dqfd: q %s / next_n_q %s / new_n_q_one_step %s / actions %s %s %s / done %s %s / is_expert %s / "
                         "weight %s do not match %s" %
                         (tuple(q.shape), tuple(next_n_q.shape), tuple(next_q1.shape), tuple(action.shape),
                          tuple(next_n_action.shape), tuple(next_action1.shape), tuple(done.shape),
                          tuple(done_one_step.shape), ie_shape, None if weight is None else tuple(weight.shape),
                          tuple(rows)))
    return qd, nq, nq1, act, nact, nact1, r, d, d1, w, ie


def _dqfd_gamma(gamma, cum_reward):
    if isinstance(gamma, list):
        raise NotImplementedError("dqfd: a list gamma (the NGU per-sample form) is not supported; no policy passes one")
    if isinstance(gamma, float) or (cum_reward and isinstance(gamma, int)):  # nstep_return takes floats only (td.py:284)
        return float(gamma)
    raise TypeError("The type of gamma should be float or list")


def _dqfd(data, gamma, lambda_n_step_td, lambda_supervised_loss, lambda_one_step_td, margin_function, nstep, cum_reward,
          value_gamma, criterion, rescale, trans_fn=None, inv_trans_fn=None):
    q, next_n_q, action, next_n_action, reward, done, done_one_step, weight, next_q1, next_action1, is_expert = data
    assert len(action.shape) == 1, action.shape  # td.py:933 / :1031
    gamma = _dqfd_gamma(gamma, cum_reward)
    if not cum_reward:
        assert reward.shape[0] == nstep  # td.py:257
    if q.dim() != 2:
        raise ValueError("dqfd: q must be (B, N), got %s" % (tuple(q.shape), ))
    B, N = q.shape
    if tuple(reward.shape) != ((B, ) if cum_reward else (nstep, B)):
        raise ValueError("dqfd: reward %s does not match B=%d, nstep=%d, cum_reward=%s" %
                         (tuple(reward.shape), B, nstep, cum_reward))
    host_out = not q.is_cuda
    dev = ops.compute_device(q, next_n_q, next_q1)
    qd, nq, nq1, act, nact, nact1, r, d, d1, w, ie = _dqfd_operands(data, B, dev, (B, ))
    compiling = torch.compiler.is_compiling()
    vg, vg_stride = (_value_gamma_op_arg if compiling else _value_gamma_arg)(value_gamma, B, dev)
    custom_trans = rescale and (trans_fn is not value_transform or inv_trans_fn is not value_inv_transform)
    code = _criterion_code(criterion)
    lam_n, lam_1, lam_s = float(lambda_n_step_td), float(lambda_one_step_td), float(lambda_supervised_loss)

    def kernel(nq_, nq1_, resc, crit, param, want_targets):
        return (torch_ops.dqfd if compiling else ops.DQfDTDFunction.apply)(
            qd, nq_, nq1_, act, nact, nact1, r, d, d1, w, vg, vg_stride, ie, B, N, int(nstep), gamma,
            1 if cum_reward else 0, resc, 1e-2, crit, param, lam_n, lam_1, lam_s, float(margin_function), 0, 0.0,
            want_targets, False)

    if code is not None and not custom_trans:
        loss, per, s_n, s_1, s_je, _, _, _ = kernel(nq, nq1, 1 if rescale else 0, code[0], code[1], False)
    else:
        # user-supplied transforms / criterion are torch callables: the kernel computes the margin term and the detached
        # targets (of the inverse-transformed next values), the callables run on the device around them
        if custom_trans:
            def inv(x, a):  # inv_trans_fn of the selected entries, at the same place of the row (td.py:1039, :1042)
                sel = a.reshape(B, 1)
                return torch.zeros_like(x).scatter_(1, sel, inv_trans_fn(x.gather(1, sel).reshape(B)).reshape(B, 1))

            nq, nq1 = inv(nq, nact), inv(nq1, nact1)
        loss_je, per_je, _, _, s_je, tn, t1, _ = kernel(nq, nq1, 1 if rescale and not custom_trans else 0, -1, 0.0, True)
        if custom_trans:
            tn, t1 = trans_fn(tn), trans_fn(t1)  # td.py:1054, :1071
        q_sa = qd.gather(1, act.reshape(B, 1)).reshape(B)
        td_n = criterion(q_sa, tn.detach())
        td_1 = criterion(q_sa, t1.detach())
        loss = ((lam_n * td_n + lam_1 * td_1) * (w if w is not None else 1.0)).mean() + loss_je
        per = lam_n * td_n.abs() + lam_1 * td_1.abs() + per_je
        s_n, s_1 = td_n.mean(), td_1.mean()
    if host_out:
        loss, per, s_n, s_1, s_je = loss.cpu(), per.cpu(), s_n.cpu(), s_1.cpu(), s_je.cpu()
    return loss, per, (s_n, s_1, s_je)


def dqfd_nstep_td_error(
        data: namedtuple,
        gamma: float,
        lambda_n_step_td: float,
        lambda_supervised_loss: float,
        margin_function: float,
        lambda_one_step_td: float = 1.,
        nstep: int = 1,
        cum_reward: bool = False,
        value_gamma: Optional[torch.Tensor] = None,
        criterion: torch.nn.modules = nn.MSELoss(reduction='none'),
) -> torch.Tensor:
    """
    DQfD loss: n-step TD + 1-step TD + supervised large-margin loss, drop-in for ding/rl_utils/td.py:870-983.

    Shapes: q, next_n_q, new_n_q_one_step (B, N); action, next_n_action, next_n_action_one_step (B,) int64; reward
    (nstep, B) -- (B,) with ``cum_reward``; done, done_one_step (B,) float multipliers; weight (B,) or None; is_expert (B,)
    float, int or bool (or a python scalar); value_gamma None, scalar, 0-dim or (B,) -- n-step target only.  gamma a float.
    As in the reference, the 1-step target uses ``reward[0]``: with ``cum_reward`` that is sample 0's reward, for every
    sample (td.py:954, :958).  Returns ``(loss, td_error_per_sample, (td_n.mean(), td_1.mean(), JE.mean()))``, all
    differentiable w.r.t. ``q``; the margin term's gradient goes to the first maximal entry of ``q + margin``.
    One forward and one backward launch.
    """
    return _dqfd(data, gamma, lambda_n_step_td, lambda_supervised_loss, lambda_one_step_td, margin_function, nstep,
                 cum_reward, value_gamma, criterion, False)


def dqfd_nstep_td_error_with_rescale(
    data: namedtuple,
    gamma: float,
    lambda_n_step_td: float,
    lambda_supervised_loss: float,
    lambda_one_step_td: float,
    margin_function: float,
    nstep: int = 1,
    cum_reward: bool = False,
    value_gamma: Optional[torch.Tensor] = None,
    criterion: torch.nn.modules = nn.MSELoss(reduction='none'),
    trans_fn: Callable = value_transform,
    inv_trans_fn: Callable = value_inv_transform,
) -> torch.Tensor:
    """
    DQfD loss with value rescaling h / h^-1 on both targets, drop-in for ding/rl_utils/td.py:986-1090.  Note the
    parameter order, kept from the reference: ``lambda_one_step_td`` comes before ``margin_function`` here, after it in
    ``dqfd_nstep_td_error``.  With the default transforms everything runs in one kernel.
    """
    return _dqfd(data, gamma, lambda_n_step_td, lambda_supervised_loss, lambda_one_step_td, margin_function, nstep,
                 cum_reward, value_gamma, criterion, True, trans_fn, inv_trans_fn)


def dqfd_nstep_td_error_sequence(
        data: namedtuple,
        gamma: float,
        lambda_n_step_td: float,
        lambda_supervised_loss: float,
        margin_function: float,
        lambda_one_step_td: float = 1.,
        nstep: int = 1,
        value_gamma: Optional[torch.Tensor] = None,
        rescale: bool = False,
        priority_mix: float = 0.9,
        criterion: torch.nn.modules = nn.MSELoss(reduction='none'),
):
    """
    R2D3's per-time-step loop over the DQfD loss in ONE launch.  Not a reference function: it is what
    ``R2D3Policy._forward_learn`` computes around the operator (ding/policy/r2d3.py:322-388)::

        for t in range(T):
            l, e, s = dqfd_nstep_td_error[_with_rescale](dqfd_nstep_td_data(q[t], ..., is_expert[t]), gamma, ...,
                                                         nstep, False, value_gamma=value_gamma[t])
            loss.append(l); td_error.append(e); stats.append(s)
        loss = sum(loss) / (len(loss) + 1e-8)          # and each of the three statistics alike
        priority = mix * max_t(td_error) + (1 - mix) * sum_t(td_error) / (len(td_error) + 1e-8)   # no abs

    The parameters are named as in ``dqfd_nstep_td_error``.  R2D3 passes the same positional list to both reference
    functions (r2d3.py:340-370), and ``dqfd_nstep_td_error_with_rescale`` takes ``lambda_one_step_td`` before
    ``margin_function``: with ``value_rescale`` on, R2D3's margin lands in ``lambda_one_step_td`` and its one-step weight
    in ``margin_function``.  This function does not swap anything; to reproduce R2D3 with rescale, pass
    ``margin_function=policy.lambda_one_step_td, lambda_one_step_td=policy.margin_function``.

    Shapes: q, next_n_q, new_n_q_one_step (T, B, N); action, next_n_action, next_n_action_one_step, done, done_one_step,
    is_expert (T, B); weight (T, B) or None; reward (T, nstep, B) (the policy's permuted layout, r2d3.py:316); value_gamma
    (T, B) or None.  Returns ``(loss, priority (B,), td_error (T, B), (loss_n, loss_1, loss_sl))``: everything but the
    priority carries gradient to ``q``.
    """
    q, next_n_q, action, next_n_action, reward, done, done_one_step, weight, next_q1, next_action1, is_expert = data
    if q.dim() != 3 or action.dim() != 2 or reward.dim() != 3:
        raise ValueError("dqfd_nstep_td_error_sequence: expected q (T, B, N), action (T, B), reward (T, nstep, B); got %s "
                         "/ %s / %s" % (tuple(q.shape), tuple(action.shape), tuple(reward.shape)))
    T, B, N = q.shape
    assert reward.shape[1] == nstep  # td.py:257 for every step
    gamma = _dqfd_gamma(gamma, False)
    code = _criterion_code(criterion)
    if code is None:
        raise NotImplementedError("dqfd_nstep_td_error_sequence: criterion must be MSELoss / L1Loss / SmoothL1Loss / "
                                  "HuberLoss with reduction='none'")
    if tuple(reward.shape) != (T, nstep, B):
        raise ValueError("dqfd_nstep_td_error_sequence: reward %s does not match T=%d, nstep=%d, B=%d" %
                         (tuple(reward.shape), T, nstep, B))
    host_out = not q.is_cuda
    dev = ops.compute_device(q, next_n_q, next_q1)
    S = T * B
    if weight is not None and weight.numel() != S:
        weight = weight.expand(T, B)
    qd, nq, nq1, act, nact, nact1, r, d, d1, w, ie = _dqfd_operands(
        dqfd_nstep_td_data(q, next_n_q, action, next_n_action, reward, done, done_one_step, weight, next_q1, next_action1,
                           is_expert), S, dev, (T, B))
    compiling = torch.compiler.is_compiling()
    vg, vg_stride = (_value_gamma_op_arg if compiling else _value_gamma_arg)(value_gamma, S, dev)
    loss, per, s_n, s_1, s_je, _, _, prio = (torch_ops.dqfd if compiling else ops.DQfDTDFunction.apply)(
        qd, nq, nq1, act, nact, nact1, r, d, d1, w, vg, vg_stride, ie, S, N, int(nstep), gamma, 0, 1 if rescale else 0,
        1e-2, code[0], code[1], float(lambda_n_step_td), float(lambda_one_step_td), float(lambda_supervised_loss),
        float(margin_function), T, float(priority_mix), False, True
    )
    per = per.reshape(T, B)
    if host_out:
        loss, prio, per, s_n, s_1, s_je = loss.cpu(), prio.cpu(), per.cpu(), s_n.cpu(), s_1.cpu(), s_je.cpu()
    return loss, prio, per, (s_n, s_1, s_je)


m_q_1step_td_data = namedtuple('m_q_1step_td_data', ['q', 'target_q', 'next_q', 'act', 'reward', 'done', 'weight'])
q_v_1step_td_data = namedtuple('q_v_1step_td_data', ['q', 'v', 'act', 'reward', 'done', 'weight'])


def _soft_done(done, dev):
    """``done`` as the float multiplier of ``(1 - done)``; a bool tensor raises as the reference's ``1 - done`` does"""
    if done.dtype == torch.bool:
        raise RuntimeError("Subtraction, the `-` operator, with a bool tensor is not supported. If you are trying to invert a "
                           "mask, use the `~` or `logical_not()` operator instead.")
    return ops.f32c(ops.to_device(done.detach(), dev), 'done')


def _soft_weight(weight, td_shape, dev):
    """``(td_error_per_sample * weight).mean()``: a weight that broadcasts to the error's shape, expanded to one per row"""
    if weight is None:
        return None
    w = ops.f32c(ops.to_device(weight.detach(), dev), 'weight')
    if torch.broadcast_shapes(tuple(w.shape), tuple(td_shape)) != tuple(td_shape):
        raise ValueError("weight %s does not broadcast to the td error shape %s" % (tuple(weight.shape), tuple(td_shape)))
    return w.expand(td_shape).reshape(-1).contiguous()


def _soft_td(mode, q, target_q, next_q, act, reward, done, weight, S, G, gamma, criterion, nstep=1, tau=0.0, alpha=0.0,
             cum_reward=False, value_gamma=None):
    """The three losses on the soft_td kernel: q (S*G, N) on the compute device, carrying its gradient; the other operands
    staged there and detached.  -> (loss, td (S*G,), action_gap, clipfrac (S*G,), record_target_v (S*G,)), the last three
    empty where the mode has none."""
    R, N = q.shape
    compiling = torch.compiler.is_compiling()
    vg, vg_stride = (_value_gamma_op_arg if compiling else _value_gamma_arg)(value_gamma, S, q.device)
    code = _criterion_code(criterion)

    def kernel(q_, crit, param):
        return (torch_ops.soft_td if compiling else ops.SoftTDFunction.apply)(
            q_, target_q, next_q, act, reward, done, weight, vg, vg_stride, mode, S, G, N, int(nstep), float(gamma),
            float(tau), float(alpha), 1 if cum_reward else 0, crit, param)

    if code is not None:
        loss, per, _, gap, clip, rec = kernel(q, code[0], code[1])
        return loss, per, gap, clip, rec
    # a criterion the kernel does not know runs as torch ops on the kernel's detached target
    _, _, target, gap, clip, rec = kernel(q.detach(), 0, 0.0)
    per = criterion(q.gather(1, act.reshape(R, 1)).reshape(R), target)
    loss = (per * (weight if weight is not None else 1.0)).mean()
    return loss, per, gap, clip, rec


def m_q_1step_td_error(
        data: namedtuple,
        gamma: float,
        tau: float,
        alpha: float,
        criterion: torch.nn.modules = nn.MSELoss(reduction='none')  # noqa
) -> torch.Tensor:
    """
    Munchausen 1-step TD error (M-DQN), drop-in for ding/rl_utils/td.py:75-158.  The target is
    ``reward + alpha*clamp(log_pi[act], -1, 1) + gamma * sum_j pi'_j * (next_q_j - tau*log pi'_j) * (1 - done)``, with
    ``log_pi`` the log-softmax policy of ``target_q / tau`` and ``pi'`` the softmax policy of ``next_q / tau``.

    Shapes: q, target_q (the target network on the current observation), next_q (B, N) with N >= 2; act (B,) int64;
    reward, done (B,); weight (B,) or None.  ``tau`` and ``alpha`` are divided by as fp32 values.  Returns ``(loss,
    td_error_per_sample (B,), action_gap, clipfrac (B, 1))``: the first two differentiable w.r.t. ``q``; ``action_gap`` is
    the mean of top-1 minus top-2 of ``target_q`` and ``clipfrac`` the per-sample float flag of a clamped ``log_pi[act]``,
    neither with gradient.  One forward and one backward launch.
    """
    q, target_q, next_q, act, reward, done, weight = data
    assert len(act.shape) == 1, act.shape        # td.py:121
    assert len(reward.shape) == 1, reward.shape  # td.py:122
    if q.dim() != 2:
        raise ValueError("m_q_1step_td_error: q must be (B, N), got %s" % (tuple(q.shape), ))
    B, N = q.shape
    if N < 2:
        raise RuntimeError("selected index k out of range")  # target_q.topk(2), td.py:152
    host_out = not q.is_cuda
    dev = ops.compute_device(q, target_q, next_q)
    qd = ops.f32c(ops.to_device(q, dev), 'q')
    tq = ops.f32c(ops.to_device(target_q.detach(), dev), 'target_q')
    nq = ops.f32c(ops.to_device(next_q.detach(), dev), 'next_q')
    a = ops.i64c(ops.to_device(act, dev), N, 'act')
    r = ops.f32c(ops.to_device(reward.detach(), dev), 'reward')
    d = _soft_done(done, dev)
    if tq.shape != qd.shape or nq.shape != qd.shape or a.numel() != B or r.numel() != B or d.numel() != B:
        raise ValueError("m_q_1step_td_error: q %s / target_q %s / next_q %s / act %s / reward %s / done %s do not match" %
                         (tuple(q.shape), tuple(target_q.shape), tuple(next_q.shape), tuple(act.shape),
                          tuple(reward.shape), tuple(done.shape)))
    w = _soft_weight(weight, (B, ), dev)
    loss, per, gap, clip, _ = _soft_td(0, qd, tq, nq, a, r, d, w, B, 1, gamma, criterion, tau=tau, alpha=alpha)
    clip = clip.reshape(B, 1)
    if host_out:
        loss, per, gap, clip = loss.cpu(), per.cpu(), gap.cpu(), clip.cpu()
    return loss, per, gap, clip


def q_nstep_sql_td_error(
        data: namedtuple,
        gamma: float,
        alpha: float,
        nstep: int = 1,
        cum_reward: bool = False,
        value_gamma: Optional[torch.Tensor] = None,
        criterion: torch.nn.modules = nn.MSELoss(reduction='none'),
) -> torch.Tensor:
    """
    Soft Q-learning n-step TD error (SQL), drop-in for ding/rl_utils/td.py:1175-1245: the n-step return (td.py:230-286) of
    the soft state value ``alpha * logsumexp(next_n_q / alpha)``, with +inf replaced by 20 and -inf by -20.

    Shapes: q, next_n_q (B, N); action (B,) int64 (next_n_action is not used, as in the reference); reward (nstep, B), or
    (B,) with ``cum_reward``; done (B,); weight (B,) or None; value_gamma None, scalar, 0-dim or (B,); gamma a float (an int
    too with ``cum_reward``).  With ``cum_reward`` a (K, B) reward broadcasts the error to (K, B), as the reference's own test
    does (tests/test_td.py:449-454).  ``alpha`` is divided by as an fp32 value.  Returns ``(loss, td_error_per_sample,
    record_target_v (B,))``; ``record_target_v`` is the soft value before the return is formed, without gradient.
    """
    q, next_n_q, action, next_n_action, reward, done, weight = data
    assert len(action.shape) == 1, action.shape  # td.py:1220
    if isinstance(gamma, list):
        raise NotImplementedError("q_nstep_sql_td_error: a list gamma (the NGU per-sample form) is not supported; no policy "
                                  "passes one")
    if not (isinstance(gamma, float) or (cum_reward and isinstance(gamma, int))):
        raise TypeError("The type of gamma should be float or list")  # nstep_return, td.py:284
    if not cum_reward:
        assert reward.shape[0] == nstep  # td.py:257
    if q.dim() != 2:
        raise ValueError("q_nstep_sql_td_error: q must be (B, N), got %s" % (tuple(q.shape), ))
    B, N = q.shape
    host_out = not q.is_cuda
    dev = ops.compute_device(q, next_n_q)
    qd = ops.f32c(ops.to_device(q, dev), 'q')
    nq = ops.f32c(ops.to_device(next_n_q.detach(), dev), 'next_n_q')
    a = ops.i64c(ops.to_device(action, dev), N)
    r = ops.f32c(ops.to_device(reward.detach(), dev), 'reward')
    d = _soft_done(done, dev)
    if nq.shape != qd.shape or a.numel() != B or d.numel() != B:
        raise ValueError("q_nstep_sql_td_error: q %s / next_n_q %s / action %s / done %s do not match" %
                         (tuple(q.shape), tuple(next_n_q.shape), tuple(action.shape), tuple(done.shape)))
    td_shape = (B, )
    vg = value_gamma
    if cum_reward and r.dim() == 2 and r.shape[1] == B:
        # reward + v * target_v * (1 - done) broadcasts to (K, B) (td.py:1239-1241): K independent row sets of the same q
        K = r.shape[0]
        td_shape = (K, B)

        def rep(x):
            return x.unsqueeze(0).expand((K, ) + tuple(x.shape)).reshape((K * B, ) + tuple(x.shape[1:]))

        qd, nq, a, d = rep(qd), rep(nq), rep(a), rep(d)
        r = r.reshape(K * B)
        if isinstance(vg, torch.Tensor) and vg.numel() == B:
            vg = rep(ops.to_device(vg.detach(), dev).reshape(B))
    elif tuple(r.shape) != ((B, ) if cum_reward else (nstep, B)):
        raise ValueError("q_nstep_sql_td_error: reward %s does not match B=%d, nstep=%d, cum_reward=%s" %
                         (tuple(reward.shape), B, nstep, cum_reward))
    w = _soft_weight(weight, td_shape, dev)
    S = qd.shape[0]
    loss, per, _, _, rec = _soft_td(1, qd, None, nq, a, r, d, w, S, 1, gamma, criterion, nstep=nstep, alpha=alpha,
                                    cum_reward=cum_reward, value_gamma=vg)
    per, rec = per.reshape(td_shape), rec[:B]
    if host_out:
        loss, per, rec = loss.cpu(), per.cpu(), rec.cpu()
    return loss, per, rec


def q_v_1step_td_error(
        data: namedtuple, gamma: float, criterion: torch.nn.modules = nn.MSELoss(reduction='none')
) -> torch.Tensor:
    """
    1-step TD error between q and a state value (the discrete SAC critic), drop-in for ding/rl_utils/td.py:161-219:
    ``target = gamma * (1 - done) * v + reward``.

    Shapes: q (B, N), act (B,) int64, v (B,); or the multi-agent form q (B, A, N), act (B, A), v (B, A), whose reward and
    done are broadcast over the A agents.  reward, done (B,); weight None or broadcastable to the error's shape.  Returns
    ``(loss, td_error_per_sample)``, the error shaped like ``act``; both differentiable w.r.t. ``q``.
    """
    q, v, act, reward, done, weight = data
    assert len(reward.shape) == 1, reward.shape  # td.py:200 / :207
    if act.dim() == 1:
        B, A = act.shape[0], 1
    elif act.dim() == 2:
        B, A = act.shape
    else:
        raise ValueError("q_v_1step_td_error: act must be (B,) or (B, A), got %s" % (tuple(act.shape), ))
    td_shape = tuple(act.shape)
    N = q.shape[-1]
    if tuple(q.shape) != td_shape + (N, ) or tuple(v.shape) != td_shape:
        raise ValueError("q_v_1step_td_error: q %s / v %s do not match act %s" %
                         (tuple(q.shape), tuple(v.shape), tuple(act.shape)))
    host_out = not q.is_cuda
    dev = ops.compute_device(q, v)
    qd = ops.f32c(ops.to_device(q, dev), 'q').reshape(B * A, N)
    vv = ops.f32c(ops.to_device(v.detach(), dev), 'v')
    a = ops.i64c(ops.to_device(act, dev), N, 'act')
    r = ops.f32c(ops.to_device(reward.detach(), dev), 'reward')
    d = _soft_done(done, dev)
    if r.numel() != B or d.numel() != B:
        raise ValueError("q_v_1step_td_error: reward %s / done %s do not match B=%d" %
                         (tuple(reward.shape), tuple(done.shape), B))
    w = _soft_weight(weight, td_shape, dev)
    loss, per, _, _, _ = _soft_td(2, qd, None, vv, a, r, d, w, B, A, gamma, criterion)
    per = per.reshape(td_shape)
    if host_out:
        loss, per = loss.cpu(), per.cpu()
    return loss, per


def _as_columns(v, next_v, reward, done, weight, value_gamma=None, nstep=None):
    """State values as a one-action Q table: (S, 1) q / next_q with action 0, per-sample tensors flattened to S = v.numel().
    ``reward``/``done``/``value_gamma`` of shape (B,) against v (B, K) are repeated along K like the reference's
    ``unsqueeze(1)`` broadcast (td.py:563-567)."""
    dev = ops.compute_device(v, next_v)
    S = v.numel()

    def per_sample(x, lead=0):
        if x is None:
            return None
        x = ops.to_device(x.detach() if isinstance(x, torch.Tensor) else x, dev)
        if x.dim() - lead < v.dim():  # (B,) against (B, K): broadcast over the trailing dims of v
            x = x.reshape(tuple(x.shape) + (1, ) * (v.dim() - (x.dim() - lead))).expand(tuple(x.shape[:lead]) + tuple(v.shape))
        return x.reshape(tuple(x.shape[:lead]) + (S, ))

    zero = torch.zeros(S, dtype=torch.int64, device=dev)
    r = per_sample(reward, lead=0 if nstep is None else 1)
    if nstep is None:
        r = r.unsqueeze(0)
    d = per_sample(done)
    if d is None:
        d = torch.zeros(S, dtype=torch.float32, device=dev)
    if weight is not None and not isinstance(weight, torch.Tensor):
        weight = ops.const_scalar(weight, dev).expand(S)  # a python-float weight (tests/test_td.py:389) scales every sample
    w = per_sample(weight)
    vg = value_gamma
    if isinstance(vg, torch.Tensor) and vg.numel() > 1:
        vg = per_sample(vg)
    return q_nstep_td_data(ops.to_device(v, dev).reshape(S, 1), ops.to_device(next_v.detach(), dev).reshape(S, 1), zero,
                           zero, r, d, w), vg


def v_1step_td_error(
        data: namedtuple,
        gamma: float,
        criterion: torch.nn.modules = nn.MSELoss(reduction='none'),
) -> torch.Tensor:
    """
    1-step TD error for a state-value (or critic) head, drop-in for ding/rl_utils/td.py:529-573 -- the critic loss of
    DDPG / TD3 / SAC / ...: ``target = gamma*(1-done)*next_v + reward``.  v, next_v (B,) or (B, K) with reward, done (B,)
    broadcast over K; done and weight may be None.  Returns ``(loss, td_error_per_sample)`` (the latter detached and
    shaped like ``v``).  Runs on the q-n-step kernel with one action column.
    """
    v, next_v, reward, done, weight = data
    host_out = not v.is_cuda
    qd, _ = _as_columns(v, next_v, reward, done, weight)
    loss, per = _qntd(qd, gamma, 1, False, None, criterion, False)
    per = per.reshape(v.shape)
    if host_out:
        loss, per = loss.cpu(), per.cpu()
    return loss, per


def v_nstep_td_error(
        data: namedtuple,
        gamma: float,
        nstep: int = 1,
        criterion: torch.nn.modules = nn.MSELoss(reduction='none'),
) -> torch.Tensor:
    """
    n-step TD error for a state-value head, drop-in for ding/rl_utils/td.py:579-617: ``target = nstep_return(reward,
    next_n_v, done, gamma, nstep, value_gamma)``.  v, next_n_v, done (B,); reward (nstep, B); weight, value_gamma (B,) or
    None.  Returns ``(loss, td_error_per_sample)``.  Runs on the q-n-step kernel with one action column.
    """
    v, next_n_v, reward, done, weight, value_gamma = data
    host_out = not v.is_cuda
    qd, vg = _as_columns(v, next_n_v, reward, done, weight, value_gamma, nstep=nstep)
    loss, per = _qntd(qd, gamma, nstep, False, vg, criterion, False)
    per = per.reshape(v.shape)
    if host_out:
        loss, per = loss.cpu(), per.cpu()
    return loss, per


def _support(v_min, v_max, n_atom, dev):
    key = (float(v_min), float(v_max), int(n_atom), dev.index)
    s = _SUPPORT_CACHE.get(key)
    if s is None:
        # built on the host then moved, exactly like td.py:457 -- CPU and CUDA linspace differ in the last bit
        s = ops.lasting(lambda: torch.linspace(v_min, v_max, n_atom).to(dev), dev)
        _SUPPORT_CACHE[key] = s
    return s


def dist_nstep_td_error(
        data: namedtuple,
        gamma: float,
        v_min: float,
        v_max: float,
        n_atom: int,
        nstep: int = 1,
        value_gamma: Optional[torch.Tensor] = None,
) -> torch.Tensor:
    """
    Multi-step TD error of categorical (C51) distributional Q-learning, drop-in for ding/rl_utils/td.py:413-523.

    Shapes: dist, next_n_dist (B, N, n_atom) probabilities -- or (B, A, N, n_atom) with (B, A) actions
    (td.py:470-489); act, next_n_act (B,) int64; reward (nstep, B); done (B,); weight None, python float, 1-element
    or per-row tensor; value_gamma None, float, 0-dim or (B,) tensor.
    Returns ``(loss, td_error_per_sample)`` -- weighted mean loss, UNWEIGHTED per-sample error (td.py:519-521).
    """
    return _dntd(data, gamma, v_min, v_max, n_atom, nstep, value_gamma, check_positive=CHECK_DIST_POSITIVE)


def _dntd(data, gamma, v_min, v_max, n_atom, nstep, value_gamma, check_positive):
    dist, next_n_dist, act, next_n_act, reward, done, weight = data
    dev = ops.compute_device(dist, next_n_dist)
    host_out = not dist.is_cuda
    if act.dim() == 1:
        B, A = act.shape[0], 1
        N = dist.shape[1]
    else:
        B, A = act.shape
        N = dist.shape[2]
    R = B * A
    if dist.shape[-1] != n_atom or dist.numel() != R * N * n_atom or next_n_dist.numel() != dist.numel():
        raise ValueError("dist %s does not match act %s / n_atom=%d" % (tuple(dist.shape), tuple(act.shape), n_atom))
    assert reward.shape[0] == nstep and reward.numel() == nstep * B, reward.shape
    dd = ops.f32c(ops.to_device(dist, dev), 'dist')
    nd = ops.f32c(ops.to_device(next_n_dist.detach(), dev), 'next_n_dist')
    a = ops.i64c(ops.to_device(act, dev), N, 'act')
    na = ops.i64c(ops.to_device(next_n_act, dev), N, 'next_n_act')
    r = ops.f32c(ops.to_device(reward.detach(), dev), 'reward')
    d = ops.f32c(ops.to_device(done.detach(), dev), 'done')
    if weight is None:
        w, w_stride = None, 0
    elif not isinstance(weight, torch.Tensor):
        w, w_stride = (float(weight) if torch.compiler.is_compiling() else ops.const_scalar(weight, dev)), 0
    else:
        w = ops.f32c(ops.to_device(weight.detach(), dev), 'weight')
        if w.numel() == 1:
            w, w_stride = w.reshape(1), 0
        elif w.numel() == R:
            w, w_stride = w.reshape(R), 1
        else:
            raise ValueError("weight must have 1 or %d elements, got %s" % (R, tuple(weight.shape)))
    if torch.compiler.is_compiling():
        vg, vg_stride = _value_gamma_op_arg(value_gamma, B, dev)
        loss, per = torch_ops.dist_nstep_td(dd, nd, a, na, r, d, w, w_stride, vg, vg_stride, B, A, N, int(n_atom),
                                            int(nstep), float(gamma), float(v_min), float(v_max), check_positive)
        return (loss.cpu(), per.cpu()) if host_out else (loss, per)
    vg, vg_stride = _value_gamma_arg(value_gamma, B, dev)
    bad = torch.zeros(1, dtype=torch.int32, device=dev) if check_positive else None
    loss, per = ops.DistNStepTDFunction.apply(
        dd, nd, a, na, r, d, w, w_stride, vg, vg_stride, _support(v_min, v_max, n_atom, dev), B, A, N, int(n_atom),
        int(nstep), float(gamma), float(v_min), float(v_max), bad
    )
    if check_positive:
        assert bad.item() == 0, ("dist act", "non-positive probability in dist[batch_range, act]")  # td.py:513
    if host_out:
        loss, per = loss.cpu(), per.cpu()
    return loss, per


def dist_1step_td_error(
        data: namedtuple,
        gamma: float,
        v_min: float,
        v_max: float,
        n_atom: int,
) -> torch.Tensor:
    """
    1-step TD error of categorical (C51) distributional Q-learning, drop-in for ding/rl_utils/td.py:294-383: the
    ``nstep = 1`` case of ``dist_nstep_td_error`` (the reference pins that identity, tests/test_td.py:272-289) on the same
    kernel, returning the loss only.  dist, next_dist (B, N, n_atom) -- or (B, A, N, n_atom) with (B, A) actions; reward,
    done (B,); weight None (or a (B, 1) / 1-element tensor).  Unlike the n-step form the reference does not assert
    ``dist > 0`` here, so neither does this.
    """
    dist, next_dist, act, next_act, reward, done, weight = data
    assert len(reward.shape) == 1, reward.shape  # td.py:343
    if isinstance(weight, torch.Tensor) and weight.dim() == 2 and weight.shape[-1] == 1:
        weight = weight.squeeze(-1)
    loss, _ = _dntd(dist_nstep_td_data(dist, next_dist, act, next_act, reward.unsqueeze(0), done, weight), gamma, v_min,
                    v_max, n_atom, 1, None, check_positive=False)
    return loss


def _lambda_operand(x, like, dev, name):
    """gammas / lambda_ / done operand of the lambda-return: python scalar -> (None, scalar, False); tensor -> ((T,B), 0, rg)
    where rg says whether gradient has to flow back into it."""
    if x is None:
        return None, 0.0, False
    if not isinstance(x, torch.Tensor):
        return None, float(x), False
    rg = x.requires_grad and x.dtype.is_floating_point and torch.is_grad_enabled()
    t = ops.to_device(x if rg else x.detach(), dev)
    t = ops.f32c(t, name)
    if t.shape != like.shape:
        t = t.expand_as(like).contiguous()
    return t, 0.0, rg


def generalized_lambda_returns(
        bootstrap_values: torch.Tensor,
        rewards: torch.Tensor,
        gammas: float,
        lambda_: float,
        done: Optional[torch.Tensor] = None
) -> torch.Tensor:
    """
    Lambda-return G_t = r_t + (1-d_t)(gamma_t lambda_t G_{t+1} + gamma_t (1-lambda_t) V_{t+1}), drop-in for
    ding/rl_utils/td.py:1574-1651.  bootstrap_values (T+1, B); rewards (T, B) -- any trailing dims are accepted, e.g.
    Dreamer's (H, B, 1) (mbpolicy/utils.py:75); gammas / lambda_ floats or tensors shaped like rewards (bool lambdas as
    produced by UPGO are accepted); done None or shaped like rewards.  The forward values are bit-exact; like the
    reference function (plain torch arithmetic) the result is differentiable: gradients reach bootstrap_values, rewards
    and tensor gammas / lambda_ that require grad (MBSAC's actor loss back-propagates through it, mbpolicy/mbsac.py:137,153)
    through one transposed-scan launch.
    """
    dev = ops.compute_device(bootstrap_values, rewards)
    host_out = not bootstrap_values.is_cuda
    grad_on = torch.is_grad_enabled()
    rg_v = bootstrap_values.requires_grad and grad_on
    rg_r = rewards.requires_grad and grad_on
    v = ops.f32c(ops.to_device(bootstrap_values if rg_v else bootstrap_values.detach(), dev), 'bootstrap_values')
    r = ops.f32c(ops.to_device(rewards if rg_r else rewards.detach(), dev), 'rewards')
    if v.dim() < 1 or v.dim() != r.dim() or v.shape[0] != r.shape[0] + 1 or v.shape[1:] != r.shape[1:]:
        raise ValueError("expected bootstrap_values (T+1, B) and rewards (T, B), got %s / %s" %
                         (tuple(v.shape), tuple(r.shape)))
    out_shape = r.shape
    T = r.shape[0]
    v, r = v.reshape(T + 1, -1), r.reshape(T, -1)  # (T, B, ...) -> (T, B'): every trailing element is its own column

    def flat(x):
        return x.reshape(T, -1) if isinstance(x, torch.Tensor) and x.dim() == len(out_shape) else x

    gt, gs, rg_g = _lambda_operand(flat(gammas), r, dev, 'gammas')
    lt, ls, rg_l = _lambda_operand(flat(lambda_), r, dev, 'lambda_')
    dt = None
    if isinstance(done, torch.Tensor):
        dt, _, _ = _lambda_operand(flat(done.detach()), r, dev, 'done')
    elif done is not None:
        dt = torch.full_like(r, float(done))
    if rg_v or rg_r or rg_g or rg_l:
        ret = ops.LambdaReturnsFunction.apply(v, r, gt, lt, dt, gs, ls, False)
    else:
        ret = ops.lambda_returns_(v, r, gt, gs, lt, ls, dt, False)
    ret = ret.reshape(out_shape)
    return ret.cpu() if host_out else ret


def td_lambda_error(data: namedtuple, gamma: float = 0.9, lambda_: float = 0.8) -> torch.Tensor:
    """
    TD(lambda) loss 0.5 * mean(w * (G^lambda - V_{:-1})^2), drop-in for ding/rl_utils/td.py:1539-1571.
    value (T+1, B) (gradient reaches value[:-1]); reward (T, B); weight None or broadcastable to (T, B).
    Scan and loss head run in one kernel.
    """
    value, reward, weight = data
    dev = ops.compute_device(value, reward)
    host_out = not value.is_cuda
    v = ops.f32c(ops.to_device(value, dev), 'value')
    r = ops.f32c(ops.to_device(reward.detach(), dev), 'reward')
    if v.dim() != 2 or r.dim() != 2 or v.shape[0] != r.shape[0] + 1 or v.shape[1] != r.shape[1]:
        raise ValueError("expected value (T+1, B) and reward (T, B), got %s / %s" % (tuple(v.shape), tuple(r.shape)))
    w = None
    if weight is not None:
        w = ops.f32c(ops.to_device(weight.detach(), dev), 'weight')
        if w.shape != r.shape:
            w = w.expand_as(r).contiguous()
    if torch.compiler.is_compiling():
        loss = torch_ops.td_lambda(v, r, w, float(gamma), float(lambda_))
    else:
        loss = ops.td_lambda_(v, r, w, gamma, lambda_)
    return loss.cpu() if host_out else loss
