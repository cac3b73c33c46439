"""``coma_error`` with the signature and namedtuples of ding/rl_utils/coma.py:6-58 -- csrc/td.cu (lambda-return scan, COMA
head) + csrc/pg.cu (policy row head)."""
from collections import namedtuple

import torch

from .. import ops, torch_ops

coma_data = namedtuple('coma_data', ['logit', 'action', 'q_value', 'target_q_value', 'reward', 'weight'])
coma_loss = namedtuple('coma_loss', ['policy_loss', 'q_value_loss', 'entropy_loss'])


def coma_error(data: namedtuple, gamma: float, lambda_: float) -> namedtuple:
    """
    COMA loss, drop-in for ding/rl_utils/coma.py:10-58.  logit, q_value, target_q_value (T, B, A, N); action (T, B, A) int64;
    reward (T, B), shared by the A agents; weight (T, B, A) -- or broadcastable to it with T leading -- or None.
      - ``q_value_loss = mean(w * (G - q_taken)^2)`` over rows t < T-1, with G the lambda-return of target_q_value taken at
        the action and reward[:-1] (the last reward row is never read);
      - ``policy_loss = -mean(logp * adv * w)`` and ``entropy_loss = mean(H * w)`` over all rows, with the detached
        ``adv = q_taken - sum(softmax(logit) * q_value)``.
    Three differentiable 0-dim tensors.  logit gets the policy and entropy gradients and q_value the value-loss gradient (at
    the action column of rows t < T-1).  As in the reference the returns are not detached: when target_q_value or reward
    requires grad it receives the value loss's gradient through the lambda-return (reward's summed over the agents).
    T must be at least 2: at T = 1 the reference's lambda-return indexes an empty tensor and raises IndexError, and so does
    this function.
    """
    logit, action, q_value, target_q_value, reward, weight = data
    if q_value.dim() != action.dim() + 1 or target_q_value.dim() != action.dim() + 1:
        raise RuntimeError("Index tensor must have the same number of dimensions as input tensor")  # coma.py:46 (gather)
    T, B, A = action.shape  # coma.py:48: ValueError for anything but (T, B, A)
    N = q_value.shape[-1]
    for name, t_ in (('logit', logit), ('q_value', q_value), ('target_q_value', target_q_value)):
        if tuple(t_.shape) != (T, B, A, N):
            raise ValueError("coma_error: %s %s does not match action %s and %d actions" % (name, tuple(t_.shape),
                                                                                        tuple(action.shape), N))
    if tuple(reward.shape) != (T, B):
        raise ValueError("coma_error: reward %s does not match action %s" % (tuple(reward.shape), tuple(action.shape)))
    if T < 2:
        raise IndexError("index -1 is out of bounds for dimension 0 with size 0")  # td.py:1639 on reward[:-1]
    dev = ops.compute_device(logit, q_value)
    host_out = not logit.is_cuda
    z = ops.f32c(ops.to_device(logit, dev), 'logit')
    qv = ops.f32c(ops.to_device(q_value, dev), 'q_value')
    tq = ops.f32c(ops.to_device(target_q_value, dev), 'target_q_value')
    rw = ops.f32c(ops.to_device(reward, dev), 'reward')
    act = ops.i64c(ops.to_device(action, dev), N)
    w = None
    if weight is not None:
        if weight.dim() != 3 or weight.shape[0] != T:
            raise ValueError("coma_error: weight %s does not broadcast to action %s along T" % (tuple(weight.shape),
                                                                                             tuple(action.shape)))
        w = ops.f32c(ops.to_device(weight.detach(), dev).expand(T, B, A), 'weight')
    grad_on = torch.is_grad_enabled()
    if grad_on and (tq.requires_grad or rw.requires_grad):
        # the returns take part in autograd: G again through the lambda-return's own function, which carries their gradient
        # back to the gathered target column and the agent-broadcast reward
        tq_taken = torch.gather(tq, -1, act.unsqueeze(-1)).reshape(T, B * A)
        r = rw.unsqueeze(-1).expand(T, B, A).reshape(T, B * A)[:-1].contiguous()
        ret = ops.LambdaReturnsFunction.apply(tq_taken, r, None, None, None, float(gamma), float(lambda_), False)
        p, v, e = ops.COMAFunction.apply(z, qv, tq.detach(), act, rw.detach(), w, ret, T, B, A, N, gamma, lambda_)
    elif torch.compiler.is_compiling():
        p, v, e = torch_ops.coma(z, qv, tq.detach(), act, rw.detach(), w, T, B, A, N, gamma, lambda_)
    else:
        p, v, e = ops.COMAFunction.apply(z, qv, tq.detach(), act, rw.detach(), w, None, T, B, A, N, gamma, lambda_)
    if host_out:
        p, v, e = p.cpu(), v.cpu(), e.cpu()
    return coma_loss(p, v, e)
