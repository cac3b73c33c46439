"""The hot-path launches of ``ops`` as ``torch.library`` custom ops (namespace ``b200rl``), so that ``torch.compile`` can
trace the eight operators of the reference's plugin boundary (gae, ppo_error, q_nstep_td_error,
q_nstep_td_error_with_rescale, dist_nstep_td_error, td_lambda_error, upgo_loss, vtrace_error_discrete_action) and the
language-model losses on (B, S, V) logits (grpo_policy_error, rloo_policy_error, the log-prob methods, ppo_policy_error /
ppo_error / a2c_error on token rows, ppo_value_error), the advantage recomputes (gae_returns, ppof_gae_returns,
normalize_advantage, ppo_error_adv_norm), symlog / inv_symlog, the quantile TD losses (QR-DQN, IQN, FQF) and the
continuous-action PPO losses, COMA's loss, ScatterConnection, the value-based losses of DQfD / R2D3 (dqfd_nstep_td_error,
its _with_rescale and _sequence forms), M-DQN, SQL and discrete SAC (m_q_1step_td_error, q_nstep_sql_td_error,
q_v_1step_td_error), the R2D2 / NGU loop q_nstep_td_error_sequence, FQF's fraction loss and the language-model losses
from the lm_head's hidden states (grpo / rloo / ppo_policy_error_linear, a2c_error_linear, token_logp_linear) without a
graph break, and ``mode="reduce-overhead"`` can replay a compiled learner step as a CUDA graph.

Each op's implementation is the launch function ``ops`` runs in eager mode.  ``rl_utils`` and ``torch_utils`` call the
entry points at the bottom of this module, one per operator: each runs its custom op while
``torch.compiler.is_compiling()`` and eager mode's ``autograd.Function`` (or no-grad shortcut) otherwise, and converts
the arguments the two modes take differently.  The schemas hold tensors and scalars only: the workspace, the
upstream-gradient records and cached constants are looked up inside the implementations, when the op runs.  Each
``setup_context`` reads the op's arguments by name (``_bind``) and each backward names the gradients it returns
(``_input_grads``), so neither depends on the position of an argument in the schema.

The forward-written gradients work as in eager mode, with one difference that functional ops impose: a backward op may
not return its input, so after a forward launch that wrote the gradients the backward op copies them once and runs the
verify launch on the copy (recomputing on the device when the upstream gradients differ from the record, no host sync).
At vocabulary scale that copy would cost as much as the loss: the language-model ops write no gradient in the forward op
and recompute it in the backward op from the saved per-row values, at the price of one more read of logit_new.  The
hidden-state losses keep eager's rule instead, since recomputing there would repeat the logit GEMMs: their forward op
writes dH / dW for a unit upstream gradient and the backward op scales them into fresh buffers.
"""
import functools
from types import SimpleNamespace
from typing import Optional

import torch
from torch import Tensor

from . import ops


def _empty(like):
    return like.new_empty(0)


@functools.cache
def _names(op):
    """the op's argument names, in schema order"""
    return tuple(a.name for a in op._opoverload._schema.arguments)


def _bind(op, inputs):
    """a setup_context's ``inputs`` as named fields"""
    return SimpleNamespace(**dict(zip(_names(op), inputs)))


def _input_grads(op, **grads):
    """a backward's return tuple: the named input gradients, None for every other argument"""
    assert grads.keys() <= set(_names(op)), (op, grads.keys())
    return tuple(grads.get(n) for n in _names(op))


def _unit_grad(grad_unit, other_grads, fresh):
    """ops._unit_grad's rule for the backward ops that take ``skip_if_unit``: (a copy of the forward-written gradient
    for a unit upstream gradient, 1) when the forward wrote one (a non-empty ``grad_unit``) and no gradient arrived
    through an output other than the loss; else (fresh(), 0), and the launch recomputes"""
    if grad_unit.numel() and all(g is None for g in other_grads):
        return grad_unit.clone(), 1
    return fresh(), 0


def _forward_grads(written, g_used, *grads):
    """copies of the forward-written gradients and their record, or None when the forward wrote none"""
    return tuple(g.clone() for g in grads) + (g_used, ) if written else None


def _upstream(g, n):
    """the device pointers of the first ``n`` floats of an upstream-gradient vector (None: no gradient, 0)"""
    g = None if g is None else g.float().contiguous()
    return g, tuple(None if g is None else g.data_ptr() + 4 * i for i in range(n))


def _one(g):
    g = None if g is None else g.float().contiguous()
    return g, ops.ptr(g)


# ---------------------------------------------------------------------------------------------------------------------
# gae: next_value is masked in place by (1 - done), as in eager mode and the reference
# ---------------------------------------------------------------------------------------------------------------------
@torch.library.custom_op('b200rl::gae', mutates_args=('next_value', ))
def gae_op(value: Tensor, next_value: Tensor, reward: Tensor, done: Optional[Tensor], traj_flag: Optional[Tensor],
           gamma: float, lambda_: float, agents: int) -> Tensor:
    return ops.gae_(value, next_value, reward, done, traj_flag, gamma, lambda_, agents)


@gae_op.register_fake
def _(value, next_value, reward, done, traj_flag, gamma, lambda_, agents):
    return torch.empty_like(value)


# ---------------------------------------------------------------------------------------------------------------------
# ppo_error
# ---------------------------------------------------------------------------------------------------------------------
@torch.library.custom_op('b200rl::ppo_loss', mutates_args=())
def ppo_loss(logit_new: Tensor, value_new: Tensor, logit_old: Tensor, action: Tensor, value_old: Tensor, adv: Tensor,
            return_: Tensor, weight: Optional[Tensor], logit_pre: Optional[Tensor], adv_stats: Optional[Tensor],
            factor: Optional[Tensor], S: int, G: int, N: int, clip_ratio: float, use_value_clip: int, dual_clip: float,
            kl_type: int, hint_kind: str, want_grad: bool) -> tuple[Tensor, Tensor, Tensor, Tensor]:
    """-> (the six floats the launch writes: policy, value, entropy, kl loss, approx_kl, clipfrac; grad_logit, grad_value,
    g_used); the last three are empty without ``want_grad``"""
    out, spec = ops.ppo_fwd_(logit_new, value_new, logit_old, action, value_old, adv, return_, weight, logit_pre, S, G, N,
                             clip_ratio, use_value_clip, dual_clip, kl_type, hint_kind, adv_stats, factor, want_grad)
    out = out[:6]
    if not want_grad:
        return out, _empty(out), _empty(out), _empty(out)
    if spec is None:  # the fused kernel did not take the problem: nothing written, the backward op recomputes
        spec = (torch.empty_like(logit_new), torch.empty_like(value_new), out.new_empty(4))
    return (out, ) + spec


@ppo_loss.register_fake
def _(logit_new, value_new, logit_old, action, value_old, adv, return_, weight, logit_pre, adv_stats, factor, S, G, N,
      clip_ratio, use_value_clip, dual_clip, kl_type, hint_kind, want_grad):
    out = logit_new.new_empty(6)
    if not want_grad:
        return out, _empty(out), _empty(out), _empty(out)
    return out, torch.empty_like(logit_new), torch.empty_like(value_new), out.new_empty(4)


@torch.library.custom_op('b200rl::ppo_bwd', mutates_args=())
def ppo_bwd(logit_new: Tensor, value_new: Tensor, logit_old: Tensor, action: Tensor, value_old: Tensor, adv: Tensor,
            return_: Tensor, weight: Optional[Tensor], logit_pre: Optional[Tensor], adv_stats: Optional[Tensor],
            factor: Optional[Tensor], g_out: Tensor, grad_logit: Tensor, grad_value: Tensor, g_used: Tensor, S: int,
            G: int, N: int, clip_ratio: float, use_value_clip: int, dual_clip: float, kl_type: int,
            hint_kind: str) -> tuple[Tensor, Tensor]:
    """-> (grad_logit, grad_value) for the upstream gradients g_out[0:4] of policy, value, entropy and kl loss"""
    keep, upstream = _upstream(g_out, 4)
    saved = (logit_new, value_new, logit_old, action, value_old, adv, return_, weight, logit_pre)
    cfg = (S, G, N, clip_ratio, use_value_clip, dual_clip, kl_type, ops.ptr(adv_stats), ops.ptr(factor))
    # whether ppo_loss's launch wrote the gradients: the question ops.ppo_fwd_ asked the library, about the same buffers
    written = g_used.numel() and ops.PPO_FUSED_BACKWARD and ops.lib().b200rl_ppo_fused_supported(
        *(ops.ptr(t) for t in (logit_new, logit_old, logit_pre, action, value_new, value_old, adv, return_, weight)),
        ops.ptr(grad_logit), G, N)
    return ops.ppo_bwd_(saved, cfg, upstream, _forward_grads(written, g_used, grad_logit, grad_value), hint_kind)


@ppo_bwd.register_fake
def _(logit_new, value_new, *args):
    return torch.empty_like(logit_new), torch.empty_like(value_new)


def _ppo_setup(ctx, inputs, output):
    a = _bind(ppo_loss, inputs)
    ctx.save_for_backward(a.logit_new, a.value_new, a.logit_old, a.action, a.value_old, a.adv, a.return_, a.weight,
                          a.logit_pre, a.adv_stats, a.factor, *output[1:])
    ctx.cfg = (a.S, a.G, a.N, a.clip_ratio, a.use_value_clip, a.dual_clip, a.kl_type, a.hint_kind)
    ctx.mark_non_differentiable(*output[1:])


def _ppo_backward(ctx, g_out, *_):
    if g_out is None:
        return _input_grads(ppo_loss)
    saved = ctx.saved_tensors
    grad_logit, grad_value = ppo_bwd(*saved[:11], g_out, *saved[11:], *ctx.cfg)
    return _input_grads(ppo_loss, logit_new=grad_logit, value_new=grad_value)


ppo_loss.register_autograd(_ppo_backward, setup_context=_ppo_setup)


# ---------------------------------------------------------------------------------------------------------------------
# q_nstep_td_error / q_nstep_td_error_with_rescale
# ---------------------------------------------------------------------------------------------------------------------
@torch.library.custom_op('b200rl::qntd_fwd', mutates_args=())
def qntd_fwd(q: Tensor, next_n_q: Tensor, action: Tensor, next_n_action: Tensor, reward: Tensor, done: Tensor,
             weight: Optional[Tensor], value_gamma: Optional[Tensor], value_gamma_scalar: Optional[float], vg_stride: int,
             gamma_ps: Optional[Tensor], S: int, G: int, N: int, nstep: int, gamma: float, cum_reward: int, rescale: int,
             eps: float, criterion: int, crit_param: float, group_mean: int,
             want_grad: bool) -> tuple[Tensor, Tensor, Tensor, Tensor, Tensor]:
    """-> (loss, td, dcrit, target, grad_unit); grad_unit is empty without ``want_grad``.  A python-scalar value_gamma
    comes as ``value_gamma_scalar`` and is read from a cached device constant."""
    if value_gamma_scalar is not None:
        value_gamma = ops.const_scalar(value_gamma_scalar, q.device)
    loss, td, dcrit, target, _, grad_unit = ops.qntd_fwd_(
        q, next_n_q, action, next_n_action, reward, done, weight, value_gamma, vg_stride, gamma_ps, S, G, N, nstep, gamma,
        cum_reward, rescale, eps, criterion, crit_param, group_mean, 0, 0.0, False, want_grad)
    return loss, td, dcrit, target, grad_unit if grad_unit is not None else _empty(loss)


@qntd_fwd.register_fake
def _(q, next_n_q, action, next_n_action, reward, done, weight, value_gamma, value_gamma_scalar, vg_stride, gamma_ps, S, G,
      N, nstep, gamma, cum_reward, rescale, eps, criterion, crit_param, group_mean, want_grad):
    R = S * G
    loss = q.new_empty(())
    grad_unit = q.new_empty(R, N) if want_grad else _empty(loss)
    return loss, q.new_empty(S if group_mean else R), q.new_empty(R), q.new_empty(R), grad_unit


@torch.library.custom_op('b200rl::qntd_bwd', mutates_args=())
def qntd_bwd(dcrit: Tensor, weight: Optional[Tensor], action: Tensor, g_loss: Optional[Tensor], g_td: Optional[Tensor],
             grad_unit: Tensor, S: int, G: int, N: int, group_mean: int) -> Tensor:
    """-> d / d q (S * G, N); verifies a copy of the forward-written unit gradient when only the loss has a gradient"""
    kl, pg = _one(g_loss)
    kt, ptd = _one(g_td)
    grad, skip = _unit_grad(grad_unit, (g_td, ), lambda: dcrit.new_empty(S * G, N))
    return ops.qntd_bwd_(dcrit, weight, action, pg, ptd, S, G, N, group_mean, 0, skip, grad)


@qntd_bwd.register_fake
def _(dcrit, weight, action, g_loss, g_td, grad_unit, S, G, N, group_mean):
    return dcrit.new_empty(S * G, N)


def _qntd_setup(ctx, inputs, output):
    a = _bind(qntd_fwd, inputs)
    ctx.save_for_backward(output[2], a.weight, a.action, output[4])
    ctx.cfg = (a.S, a.G, a.N, a.group_mean)
    ctx.q_shape = a.q.shape
    ctx.set_materialize_grads(False)
    ctx.mark_non_differentiable(*output[2:])


def _qntd_backward(ctx, g_loss, g_td, *_):
    if g_loss is None and g_td is None:
        return _input_grads(qntd_fwd)
    dcrit, weight, action, grad_unit = ctx.saved_tensors
    grad = qntd_bwd(dcrit, weight, action, g_loss, g_td, grad_unit, *ctx.cfg)
    return _input_grads(qntd_fwd, q=grad.view(ctx.q_shape))


qntd_fwd.register_autograd(_qntd_backward, setup_context=_qntd_setup)


# ---------------------------------------------------------------------------------------------------------------------
# q_nstep_td_error_sequence (the R2D2 / NGU loop): the q-n-step launches with seq_len = T and the priority output
# ---------------------------------------------------------------------------------------------------------------------
@torch.library.custom_op('b200rl::qntd_seq_fwd', mutates_args=())
def qntd_seq_fwd(q: Tensor, next_n_q: Tensor, action: Tensor, next_n_action: Tensor, reward: Tensor, done: Tensor,
                 weight: Optional[Tensor], value_gamma: Optional[Tensor], value_gamma_scalar: Optional[float],
                 vg_stride: int, gamma_ps: Optional[Tensor], S: int, N: int, nstep: int, gamma: float, rescale: int,
                 criterion: int, crit_param: float, seq_len: int, priority_mix: float,
                 want_grad: bool) -> tuple[Tensor, Tensor, Tensor, Tensor, Tensor]:
    """-> (loss, td, dcrit, prio (S / seq_len), grad_unit); one row per sample (G = 1), no cum_reward, eps 1e-2, as
    q_nstep_td_error_sequence calls the launch"""
    if value_gamma_scalar is not None:
        value_gamma = ops.const_scalar(value_gamma_scalar, q.device)
    loss, td, dcrit, _, prio, grad_unit = ops.qntd_fwd_(
        q, next_n_q, action, next_n_action, reward, done, weight, value_gamma, vg_stride, gamma_ps, S, 1, N, nstep, gamma,
        0, rescale, 1e-2, criterion, crit_param, 0, seq_len, priority_mix, True, want_grad)
    return loss, td, dcrit, prio, grad_unit if grad_unit is not None else _empty(loss)


@qntd_seq_fwd.register_fake
def _(q, next_n_q, action, next_n_action, reward, done, weight, value_gamma, value_gamma_scalar, vg_stride, gamma_ps, S, N,
      nstep, gamma, rescale, criterion, crit_param, seq_len, priority_mix, want_grad):
    loss = q.new_empty(())
    return (loss, q.new_empty(S), q.new_empty(S), q.new_empty(S // seq_len),
            q.new_empty(S, N) if want_grad else _empty(loss))


@torch.library.custom_op('b200rl::qntd_seq_bwd', mutates_args=())
def qntd_seq_bwd(dcrit: Tensor, weight: Optional[Tensor], action: Tensor, g_loss: Optional[Tensor],
                 g_td: Optional[Tensor], grad_unit: Tensor, S: int, N: int, seq_len: int) -> Tensor:
    """-> d / d q (S, N), as qntd_bwd with the loss averaged over the seq_len steps"""
    kl, pg = _one(g_loss)
    kt, ptd = _one(g_td)
    grad, skip = _unit_grad(grad_unit, (g_td, ), lambda: dcrit.new_empty(S, N))
    return ops.qntd_bwd_(dcrit, weight, action, pg, ptd, S, 1, N, 0, seq_len, skip, grad)


@qntd_seq_bwd.register_fake
def _(dcrit, weight, action, g_loss, g_td, grad_unit, S, N, seq_len):
    return dcrit.new_empty(S, N)


def _qntd_seq_setup(ctx, inputs, output):
    a = _bind(qntd_seq_fwd, inputs)
    ctx.save_for_backward(output[2], a.weight, a.action, output[4])
    ctx.cfg = (a.S, a.N, a.seq_len)
    ctx.q_shape = a.q.shape
    ctx.set_materialize_grads(False)
    ctx.mark_non_differentiable(*output[2:])


def _qntd_seq_backward(ctx, g_loss, g_td, *_):
    if g_loss is None and g_td is None:
        return _input_grads(qntd_seq_fwd)
    dcrit, weight, action, grad_unit = ctx.saved_tensors
    grad = qntd_seq_bwd(dcrit, weight, action, g_loss, g_td, grad_unit, *ctx.cfg)
    return _input_grads(qntd_seq_fwd, q=grad.view(ctx.q_shape))


qntd_seq_fwd.register_autograd(_qntd_seq_backward, setup_context=_qntd_seq_setup)


# ---------------------------------------------------------------------------------------------------------------------
# dqfd_nstep_td_error[_with_rescale] and the R2D3 loop (csrc/td.cu dqfd_fwd / dqfd_bwd): the three statistics leave the op
# as one (3,) tensor, unbound by the caller (a custom op's outputs may not alias each other)
# ---------------------------------------------------------------------------------------------------------------------
@torch.library.custom_op('b200rl::dqfd_fwd', mutates_args=())
def dqfd_fwd(q: Tensor, next_n_q: Tensor, next_q1: Tensor, action: Tensor, next_n_action: Tensor, next_action1: Tensor,
             reward: Tensor, done: Tensor, done1: Tensor, weight: Optional[Tensor], value_gamma: Optional[Tensor],
             value_gamma_scalar: Optional[float], vg_stride: int, is_expert: Optional[Tensor],
             is_expert_scalar: Optional[float], S: int, N: int, nstep: int, gamma: float, cum_reward: int, rescale: int,
             eps: float, criterion: int, crit_param: float, lam_n: float, lam_1: float, lam_s: float, margin: float,
             seq_len: int, priority_mix: float, want_targets: bool, want_priority: bool,
             want_grad: bool) -> tuple[Tensor, Tensor, Tensor, Tensor, Tensor, Tensor, Tensor, Tensor]:
    """-> (loss, td, stats (3,), saved (S, 4), tn, t1, prio, grad_unit); tn / t1 / prio / grad_unit are empty where not
    wanted.  A python-scalar value_gamma or is_expert comes as a float and is read from a cached device constant (is_expert
    expanded to S rows, as in eager mode)."""
    dev = q.device
    if value_gamma_scalar is not None:
        value_gamma = ops.const_scalar(value_gamma_scalar, dev)
    if is_expert_scalar is not None:
        is_expert = ops.const_scalar(is_expert_scalar, dev).expand(S).contiguous()
    out = ops.dqfd_fwd_(q, next_n_q, next_q1, action, next_n_action, next_action1, reward, done, done1, weight,
                        value_gamma, vg_stride, is_expert, S, N, nstep, gamma, cum_reward, rescale, eps, criterion,
                        crit_param, lam_n, lam_1, lam_s, margin, seq_len, priority_mix, want_targets, want_priority,
                        want_grad)
    return tuple(x if x is not None else _empty(out[0]) for x in out)


@dqfd_fwd.register_fake
def _(q, next_n_q, next_q1, action, next_n_action, next_action1, reward, done, done1, weight, value_gamma,
      value_gamma_scalar, vg_stride, is_expert, is_expert_scalar, S, N, nstep, gamma, cum_reward, rescale, eps, criterion,
      crit_param, lam_n, lam_1, lam_s, margin, seq_len, priority_mix, want_targets, want_priority, want_grad):
    loss = q.new_empty(())
    return (loss, q.new_empty(S), q.new_empty(3), q.new_empty(S, 4), q.new_empty(S if want_targets else 0),
            q.new_empty(S if want_targets else 0), q.new_empty(S // seq_len if want_priority else 0),
            q.new_empty(S, N) if want_grad else _empty(loss))


@torch.library.custom_op('b200rl::dqfd_bwd', mutates_args=())
def dqfd_bwd(saved: Tensor, weight: Optional[Tensor], action: Tensor, g_loss: Optional[Tensor], g_td: Optional[Tensor],
             g_stats: Optional[Tensor], grad_unit: Tensor, S: int, N: int, lam_n: float, lam_1: float, lam_s: float,
             seq_len: int) -> Tensor:
    """-> d / d q (S, N); verifies a copy of the forward-written unit gradient when only the loss has a gradient"""
    kl, pg = _one(g_loss)
    kt, ptd = _one(g_td)
    ks, pstats = _upstream(g_stats, 3)
    grad, skip = _unit_grad(grad_unit, (g_td, g_stats), lambda: saved.new_empty(S, N))
    return ops.dqfd_bwd_(saved, weight, action, pg, ptd, pstats, S, N, lam_n, lam_1, lam_s, seq_len, skip, grad)


@dqfd_bwd.register_fake
def _(saved, weight, action, g_loss, g_td, g_stats, grad_unit, S, N, lam_n, lam_1, lam_s, seq_len):
    return saved.new_empty(S, N)


def _dqfd_setup(ctx, inputs, output):
    a = _bind(dqfd_fwd, inputs)
    ctx.save_for_backward(output[3], a.weight, a.action, output[7])
    ctx.cfg = (a.S, a.N, a.lam_n, a.lam_1, a.lam_s, a.seq_len)
    ctx.q_shape = a.q.shape
    ctx.set_materialize_grads(False)
    ctx.mark_non_differentiable(*output[3:])


def _dqfd_backward(ctx, g_loss, g_td, g_stats, *_):
    if g_loss is None and g_td is None and g_stats is None:
        return _input_grads(dqfd_fwd)
    saved, weight, action, grad_unit = ctx.saved_tensors
    grad = dqfd_bwd(saved, weight, action, g_loss, g_td, g_stats, grad_unit, *ctx.cfg)
    return _input_grads(dqfd_fwd, q=grad.view(ctx.q_shape))


dqfd_fwd.register_autograd(_dqfd_backward, setup_context=_dqfd_setup)


# ---------------------------------------------------------------------------------------------------------------------
# m_q_1step_td_error / q_nstep_sql_td_error / q_v_1step_td_error (csrc/td.cu soft_td_fwd): every target is detached, so
# the backward is qntd_bwd over the R rows (G = 1), as SoftTDFunction's; the statistics carry no gradient
# ---------------------------------------------------------------------------------------------------------------------
@torch.library.custom_op('b200rl::soft_td_fwd', mutates_args=())
def soft_td_fwd(q: Tensor, target_q: Optional[Tensor], next_q: Tensor, action: Tensor, reward: Tensor, done: Tensor,
                weight: Optional[Tensor], value_gamma: Optional[Tensor], value_gamma_scalar: Optional[float],
                vg_stride: int, mode: int, S: int, G: int, N: int, nstep: int, gamma: float, tau: float, alpha: float,
                cum_reward: int, criterion: int,
                crit_param: float, want_grad: bool) -> tuple[Tensor, Tensor, Tensor, Tensor, Tensor, Tensor, Tensor, Tensor]:
    """-> (loss, td, dcrit, target, action_gap, clipfrac, record_target_v, grad_unit); the statistics the mode has none
    of (M-DQN: action_gap and clipfrac; SQL: record_target_v) and grad_unit without ``want_grad`` are empty"""
    if value_gamma_scalar is not None:
        value_gamma = ops.const_scalar(value_gamma_scalar, q.device)
    out = ops.soft_td_fwd_(q, target_q, next_q, action, reward, done, weight, value_gamma, vg_stride, mode, S, G, N, nstep,
                           gamma, tau, alpha, cum_reward, criterion, crit_param, want_grad)
    return tuple(x if x is not None else _empty(out[0]) for x in out)


@soft_td_fwd.register_fake
def _(q, target_q, next_q, action, reward, done, weight, value_gamma, value_gamma_scalar, vg_stride, mode, S, G, N, nstep,
      gamma, tau, alpha, cum_reward, criterion, crit_param, want_grad):
    R = S * G
    loss = q.new_empty(())
    return (loss, q.new_empty(R), q.new_empty(R), q.new_empty(R), q.new_empty(() if mode == 0 else 0),
            q.new_empty(R if mode == 0 else 0), q.new_empty(R if mode == 1 else 0),
            q.new_empty(R, N) if want_grad else _empty(loss))


def _soft_td_setup(ctx, inputs, output):
    a = _bind(soft_td_fwd, inputs)
    ctx.save_for_backward(output[2], a.weight, a.action, output[7])
    ctx.cfg = (a.S * a.G, 1, a.N, 0)  # qntd_bwd's (S, G, N, group_mean): R rows of one
    ctx.q_shape = a.q.shape
    ctx.set_materialize_grads(False)
    ctx.mark_non_differentiable(*output[2:])


def _soft_td_backward(ctx, g_loss, g_td, *_):
    if g_loss is None and g_td is None:
        return _input_grads(soft_td_fwd)
    dcrit, weight, action, grad_unit = ctx.saved_tensors
    grad = qntd_bwd(dcrit, weight, action, g_loss, g_td, grad_unit, *ctx.cfg)
    return _input_grads(soft_td_fwd, q=grad.view(ctx.q_shape))


soft_td_fwd.register_autograd(_soft_td_backward, setup_context=_soft_td_setup)


# ---------------------------------------------------------------------------------------------------------------------
# dist_nstep_td_error
# ---------------------------------------------------------------------------------------------------------------------
@torch.library.custom_op('b200rl::dntd_fwd', mutates_args=())
def dntd_fwd(dist: Tensor, next_n_dist: Tensor, act: Tensor, next_n_act: Tensor, reward: Tensor, done: Tensor,
             weight: Optional[Tensor], weight_scalar: Optional[float], w_stride: int, value_gamma: Optional[Tensor],
             value_gamma_scalar: Optional[float], vg_stride: int, B: int, A: int, N: int, n_atom: int, nstep: int,
             gamma: float, v_min: float, v_max: float, check_positive: bool,
             want_grad: bool) -> tuple[Tensor, Tensor, Tensor, Tensor]:
    """-> (loss, td, proj, grad_unit); with ``check_positive`` the reference's assertion that dist[b, act] > 0 (one 4-byte
    device-to-host read, as in eager mode)"""
    from .rl_utils.td import _support
    dev = dist.device
    if weight_scalar is not None:
        weight = ops.const_scalar(weight_scalar, dev)
    if value_gamma_scalar is not None:
        value_gamma = ops.const_scalar(value_gamma_scalar, dev)
    bad = None
    if check_positive:
        if dev.type == 'cuda' and torch.cuda.is_current_stream_capturing():
            raise ops._lib.B200RLError(
                "dist_nstep_td_error: the check that dist[b, act] > 0 reads the device and cannot run inside a CUDA graph; "
                "set di_engine_b200.rl_utils.td.CHECK_DIST_POSITIVE = False to capture it")
        bad = torch.zeros(1, dtype=torch.int32, device=dev)
    loss, td, proj, grad_unit = ops.dntd_fwd_(dist, next_n_dist, act, next_n_act, reward, done, weight, w_stride,
                                              value_gamma, vg_stride, _support(v_min, v_max, n_atom, dev), B, A, N,
                                              n_atom, nstep, gamma, v_min, v_max, bad, want_grad)
    if check_positive:
        assert bad.item() == 0, ("dist act", "non-positive probability in dist[batch_range, act]")  # td.py:513
    return loss, td, proj, grad_unit if grad_unit is not None else _empty(loss)


@dntd_fwd.register_fake
def _(dist, next_n_dist, act, next_n_act, reward, done, weight, weight_scalar, w_stride, value_gamma, value_gamma_scalar,
      vg_stride, B, A, N, n_atom, nstep, gamma, v_min, v_max, check_positive, want_grad):
    loss = dist.new_empty(())
    return loss, dist.new_empty(B * A), dist.new_empty(B * A, n_atom), (
        torch.empty_like(dist) if want_grad else _empty(loss))


@torch.library.custom_op('b200rl::dntd_bwd', mutates_args=())
def dntd_bwd(dist: Tensor, act: Tensor, proj: Tensor, weight: Optional[Tensor], weight_scalar: Optional[float],
             w_stride: int, g_loss: Optional[Tensor], g_td: Optional[Tensor], grad_unit: Tensor, R: int, N: int,
             n_atom: int) -> Tensor:
    if weight_scalar is not None:
        weight = ops.const_scalar(weight_scalar, dist.device)
    kl, pg = _one(g_loss)
    kt, ptd = _one(g_td)
    grad, skip = _unit_grad(grad_unit, (g_td, ), lambda: torch.empty_like(dist))
    return ops.dntd_bwd_(dist, act, proj, weight, w_stride, pg, ptd, R, N, n_atom, skip, grad)


@dntd_bwd.register_fake
def _(dist, *args):
    return torch.empty_like(dist)


def _dntd_setup(ctx, inputs, output):
    a = _bind(dntd_fwd, inputs)
    ctx.save_for_backward(a.dist, a.act, output[2], a.weight, output[3])
    ctx.cfg = (a.weight_scalar, a.w_stride, a.B * a.A, a.N, a.n_atom)
    ctx.set_materialize_grads(False)
    ctx.mark_non_differentiable(*output[2:])


def _dntd_backward(ctx, g_loss, g_td, *_):
    if g_loss is None and g_td is None:
        return _input_grads(dntd_fwd)
    dist, act, proj, weight, grad_unit = ctx.saved_tensors
    weight_scalar, w_stride, R, N, n_atom = ctx.cfg
    grad = dntd_bwd(dist, act, proj, weight, weight_scalar, w_stride, g_loss, g_td, grad_unit, R, N, n_atom)
    return _input_grads(dntd_fwd, dist=grad)


dntd_fwd.register_autograd(_dntd_backward, setup_context=_dntd_setup)


# ---------------------------------------------------------------------------------------------------------------------
# td_lambda_error: the forward launch writes d loss / d value for a unit upstream gradient; backward scales it
# ---------------------------------------------------------------------------------------------------------------------
@torch.library.custom_op('b200rl::td_lambda_fwd', mutates_args=())
def td_lambda_fwd(value: Tensor, reward: Tensor, weight: Optional[Tensor], gamma: float,
                  lambda_: float) -> tuple[Tensor, Tensor]:
    return ops.td_lambda_fwd_(value, reward, weight, gamma, lambda_)


@td_lambda_fwd.register_fake
def _(value, reward, weight, gamma, lambda_):
    return value.new_empty(()), torch.empty_like(value)


@torch.library.custom_op('b200rl::scale', mutates_args=())
def scale(g: Tensor, saved: Tensor) -> Tensor:
    """``g * saved`` for a one-element upstream gradient ``g``"""
    kg, pg = _one(g)
    return ops.scale_(pg, saved)


@scale.register_fake
def _(g, saved):
    return torch.empty_like(saved)


def _td_lambda_setup(ctx, inputs, output):
    ctx.save_for_backward(output[1])
    ctx.mark_non_differentiable(output[1])


def _td_lambda_backward(ctx, g_loss, _g_dvalue):
    dvalue, = ctx.saved_tensors
    return _input_grads(td_lambda_fwd, value=scale(g_loss, dvalue))


td_lambda_fwd.register_autograd(_td_lambda_backward, setup_context=_td_lambda_setup)


# ---------------------------------------------------------------------------------------------------------------------
# upgo_loss: the UPGO lambda-return scan, then the loss head
# ---------------------------------------------------------------------------------------------------------------------
@torch.library.custom_op('b200rl::lambda_returns', mutates_args=())
def lambda_returns(value: Tensor, reward: Tensor, gammas: Optional[Tensor], gamma: float, lambdas: Optional[Tensor],
                   lambda_: float, done: Optional[Tensor], upgo_mode: bool) -> Tensor:
    return ops.lambda_returns_(value, reward, gammas, gamma, lambdas, lambda_, done, upgo_mode)


@lambda_returns.register_fake
def _(value, reward, gammas, gamma, lambdas, lambda_, done, upgo_mode):
    return torch.empty_like(reward)


@torch.library.custom_op('b200rl::upgo_fwd', mutates_args=())
def upgo_fwd(logit: Tensor, action: Tensor, mask: Optional[Tensor], rho: Tensor, ret: Tensor, value: Tensor, TB: int,
             K: int, N: int, want_grad: bool) -> tuple[Tensor, Tensor, Tensor]:
    loss, adv, grad_unit = ops.upgo_fwd_(logit, action, mask, rho, ret, value, TB, K, N, want_grad)
    return loss, adv, grad_unit if grad_unit is not None else _empty(loss)


@upgo_fwd.register_fake
def _(logit, action, mask, rho, ret, value, TB, K, N, want_grad):
    loss = logit.new_empty(())
    return loss, logit.new_empty(TB), torch.empty_like(logit) if want_grad else _empty(loss)


@torch.library.custom_op('b200rl::upgo_bwd', mutates_args=())
def upgo_bwd(logit: Tensor, action: Tensor, mask: Optional[Tensor], adv: Tensor, g_loss: Tensor, grad_unit: Tensor,
             TB: int, K: int, N: int) -> Tensor:
    grad, skip = _unit_grad(grad_unit, (), lambda: torch.empty_like(logit))  # adv, the other output, is not differentiable
    kg, pg = _one(g_loss)
    return ops.upgo_bwd_(logit, action, mask, adv, pg, TB, K, N, skip, grad)


@upgo_bwd.register_fake
def _(logit, *args):
    return torch.empty_like(logit)


def _upgo_setup(ctx, inputs, output):
    a = _bind(upgo_fwd, inputs)
    ctx.save_for_backward(a.logit, a.action, a.mask, output[1], output[2])
    ctx.cfg = (a.TB, a.K, a.N)
    ctx.mark_non_differentiable(*output[1:])


def _upgo_backward(ctx, g_loss, *_):
    logit, action, mask, adv, grad_unit = ctx.saved_tensors
    return _input_grads(upgo_fwd, logit=upgo_bwd(logit, action, mask, adv, g_loss, grad_unit, *ctx.cfg))


upgo_fwd.register_autograd(_upgo_backward, setup_context=_upgo_setup)


# ---------------------------------------------------------------------------------------------------------------------
# vtrace_error_discrete_action
# ---------------------------------------------------------------------------------------------------------------------
@torch.library.custom_op('b200rl::vtrace_loss', mutates_args=())
def vtrace_loss(target_output: Tensor, value: Tensor, behaviour_output: Tensor, action: Tensor, reward: Tensor,
               weight: Optional[Tensor], gamma: float, lambda_: float, rho_clip: float, c_clip: float, rho_pg_clip: float,
               want_grad: bool) -> tuple[Tensor, Tensor, Tensor, Tensor]:
    """-> (policy, value and entropy loss, grad_logit, grad_value, g_used): the forward-written gradients and their record
    after the one-launch kernel; after the rows / scan kernels, which write no gradients, the (T, B) records of their
    backward launch (cpg, dv) at the head of grad_value and grad_logit.  All but the first are empty without
    ``want_grad``."""
    scal = (gamma, lambda_, rho_clip, c_clip, rho_pg_clip)
    out, fused, spec, cpg, dv = ops.vtrace_fwd_(target_output, value, behaviour_output, action, reward, weight, scal,
                                                want_grad)
    out = out[:3]
    if not want_grad:
        return (out, ) + (_empty(out), ) * 3
    if fused:
        return (out, ) + spec
    grad_logit, grad_value, g_used = torch.empty_like(target_output), value.new_empty(value.shape), out.new_empty(3)
    grad_value.view(-1)[:cpg.numel()].copy_(cpg.view(-1))
    grad_logit.view(-1)[:dv.numel()].copy_(dv.view(-1))
    return out, grad_logit, grad_value, g_used


@vtrace_loss.register_fake
def _(target_output, value, behaviour_output, action, reward, weight, gamma, lambda_, rho_clip, c_clip, rho_pg_clip,
      want_grad):
    out = target_output.new_empty(3)
    if not want_grad:
        return (out, ) + (_empty(out), ) * 3
    return out, torch.empty_like(target_output), value.new_empty(value.shape), out.new_empty(3)


@torch.library.custom_op('b200rl::vtrace_bwd', mutates_args=())
def vtrace_bwd(target_output: Tensor, behaviour_output: Tensor, action: Tensor, value: Tensor, reward: Tensor,
               weight: Optional[Tensor], g_out: Tensor, grad_logit: Tensor, grad_value: Tensor, g_used: Tensor,
               gamma: float, lambda_: float, rho_clip: float, c_clip: float, rho_pg_clip: float) -> tuple[Tensor, Tensor]:
    """-> (grad_logit, grad_value) for the upstream gradients g_out[0:3] of policy, value and entropy loss"""
    keep, upstream = _upstream(g_out, 3)
    # whether vtrace_loss's one-launch kernel ran: the question ops.vtrace_fwd_ asked the library, about the same buffers
    T, B = reward.shape
    fused = ops.VTRACE_FUSED and ops.lib().b200rl_vtrace_fused_supported(
        *(ops.ptr(t) for t in (target_output, behaviour_output, action, value, reward, weight)), T, B,
        target_output.shape[-1], ops.ptr(grad_logit), ops.ptr(grad_value))
    if not fused:
        n = reward.numel()
        cpg, dv = grad_value.view(-1)[:n].view(reward.shape), grad_logit.view(-1)[:n].view(reward.shape)
        return ops.vtrace_bwd_(target_output, action, weight, cpg, dv, upstream)
    saved = (target_output, behaviour_output, action, value, reward, weight)
    return ops.vtrace_verify_(saved, (gamma, lambda_, rho_clip, c_clip, rho_pg_clip), upstream,
                              _forward_grads(True, g_used, grad_logit, grad_value))


@vtrace_bwd.register_fake
def _(target_output, behaviour_output, action, value, *args):
    return torch.empty_like(target_output), value.new_empty(value.shape)


def _vtrace_setup(ctx, inputs, output):
    a = _bind(vtrace_loss, inputs)
    ctx.save_for_backward(a.target_output, a.behaviour_output, a.action, a.value, a.reward, a.weight, *output[1:])
    ctx.scal = (a.gamma, a.lambda_, a.rho_clip, a.c_clip, a.rho_pg_clip)
    ctx.mark_non_differentiable(*output[1:])


def _vtrace_backward(ctx, g_out, *_):
    if g_out is None:
        return _input_grads(vtrace_loss)
    grad_logit, grad_value = vtrace_bwd(*ctx.saved_tensors[:6], g_out, *ctx.saved_tensors[6:], *ctx.scal)
    return _input_grads(vtrace_loss, target_output=grad_logit, value=grad_value)


vtrace_loss.register_autograd(_vtrace_backward, setup_context=_vtrace_setup)


# ---------------------------------------------------------------------------------------------------------------------
# ppo_value_error: the forward launch writes d loss / d value_new for a unit upstream gradient; backward scales it
# ---------------------------------------------------------------------------------------------------------------------
@torch.library.custom_op('b200rl::ppo_value_fwd', mutates_args=())
def ppo_value_fwd(value_new: Tensor, value_old: Tensor, return_: Tensor, weight: Optional[Tensor], clip_ratio: float,
                  use_value_clip: bool, want_grad: bool) -> tuple[Tensor, Tensor]:
    """-> (loss, d loss / d value_new; empty without ``want_grad``)"""
    loss, dvalue = ops.ppo_value_fwd_(value_new, value_old, return_, weight, clip_ratio, use_value_clip, want_grad)
    return loss, dvalue if dvalue is not None else _empty(loss)


@ppo_value_fwd.register_fake
def _(value_new, value_old, return_, weight, clip_ratio, use_value_clip, want_grad):
    loss = value_new.new_empty(())
    return loss, torch.empty_like(value_new) if want_grad else _empty(loss)


def _ppo_value_setup(ctx, inputs, output):
    ctx.save_for_backward(output[1])
    ctx.mark_non_differentiable(output[1])


def _ppo_value_backward(ctx, g_loss, _g_dvalue):
    dvalue, = ctx.saved_tensors
    return _input_grads(ppo_value_fwd, value_new=scale(g_loss, dvalue))


ppo_value_fwd.register_autograd(_ppo_value_backward, setup_context=_ppo_value_setup)


# ---------------------------------------------------------------------------------------------------------------------
# The language-model losses on (B, S, V) logits (csrc/vocab.cu).  Their gradients are recomputed in the backward op from
# the per-row values the forward op saves: the forward op writes no gradient, so nothing of (B, S, V) size is copied.
# A backward op that rewrote the forward's gradient buffer in place would have to declare that buffer mutated; after
# functionalization the buffer is an input of the backward graph that nothing copies back into, and inductor does not
# reinplace such an input -- it copies it first, which is the (B, S, V) copy this design avoids.  The cost instead is one
# more read of logit_new, in the backward op.  Each op makes the kernel's 16-byte-aligned copy of an odd-offset view
# itself (ops.logits_c): a traced tensor has no address to decide it by.
# ---------------------------------------------------------------------------------------------------------------------
def _rows(x):
    """the token rows of logits (..., V), symbolic under dynamic shapes"""
    return x.numel() // x.shape[-1]


def _f32(x, n):
    return x.new_empty(n, dtype=torch.float32)


@torch.library.custom_op('b200rl::token_logp', mutates_args=())
def token_logp_op(logits: Tensor, index: Tensor) -> tuple[Tensor, Tensor]:
    """the log-prob methods: logits (rows, V) fp32 or bf16, index (rows) -> (log p(index), logsumexp), fp32 per row"""
    x = ops.logits_c(logits)
    return ops.token_logp_fwd_(ops.logit_dtype(x), x, index)


@token_logp_op.register_fake
def _(logits, index):
    return _f32(logits, logits.shape[0]), _f32(logits, logits.shape[0])


@torch.library.custom_op('b200rl::vocab_bwd', mutates_args=())
def vocab_bwd(logits: Tensor, index: Tensor, lse: Tensor, coef: Tensor, g: Optional[Tensor]) -> Tensor:
    """d / d logits = (g[0], or 1 without ``g``) * coef[row] * (onehot(index) - softmax(logits[row])), in the logits'
    dtype: the backward of ``token_logp`` (coef its upstream gradient) and of ``lm_policy_fwd`` (coef the unit
    coefficient, g the loss's upstream gradient)"""
    x = ops.logits_c(logits)
    keep, pg = _one(g)
    return ops.token_logp_bwd_(ops.logit_dtype(x), x, index, lse, coef, pg, 0, torch.empty_like(logits))


@vocab_bwd.register_fake
def _(logits, *args):
    return torch.empty_like(logits)


def _token_logp_setup(ctx, inputs, output):
    a = _bind(token_logp_op, inputs)
    ctx.save_for_backward(a.logits, a.index, output[1])
    ctx.mark_non_differentiable(output[1])


def _token_logp_backward(ctx, g_lp, _g_lse):
    logits, index, lse = ctx.saved_tensors
    return _input_grads(token_logp_op, logits=vocab_bwd(logits, index, lse, g_lp.float().contiguous(), None))


token_logp_op.register_autograd(_token_logp_backward, setup_context=_token_logp_setup)


@torch.library.custom_op('b200rl::lm_policy_fwd', mutates_args=())
def lm_policy_fwd(logit_new: Tensor, logit_old: Tensor, logit_ref: Optional[Tensor], action: Tensor, side: Tensor,
                  weight: Optional[Tensor], mode: str, clip_ratio: float, beta: float) -> tuple[Tensor, Tensor, Tensor]:
    """grpo_policy_error (``mode`` 'grpo': side = adv (B)) or rloo_policy_error ('rloo': side = reward (K, B / K)) on
    logits (B, S, V) -> (loss / approx_kl / clipfrac, logsumexp of logit_new per row, d loss / d lp_new per row for a unit
    upstream gradient)"""
    xs = [ops.logits_c(x) if x is not None else None for x in (logit_new, logit_old, logit_ref)]
    dt = ops.logit_dtype(xs[0])
    if mode == 'grpo':
        return ops.grpo_fwd_(xs[0], xs[1], xs[2], action, side, weight, dt, clip_ratio, beta, None)
    return ops.rloo_fwd_(xs[0], xs[1], action, side, weight, dt, clip_ratio, None)


@lm_policy_fwd.register_fake
def _(logit_new, logit_old, logit_ref, action, side, weight, mode, clip_ratio, beta):
    rows = logit_new.shape[0] * logit_new.shape[1]
    return _f32(logit_new, 3), _f32(logit_new, rows), _f32(logit_new, rows)


def _lm_policy_setup(ctx, inputs, output):
    a = _bind(lm_policy_fwd, inputs)
    ctx.save_for_backward(a.logit_new, a.action, output[1], output[2])
    ctx.set_materialize_grads(False)
    ctx.mark_non_differentiable(output[1], output[2])


def _lm_policy_backward(ctx, g_out, _g_lse, _g_dlp):
    if g_out is None:
        return _input_grads(lm_policy_fwd)
    logit_new, action, lse, dlp = ctx.saved_tensors
    return _input_grads(lm_policy_fwd, logit_new=vocab_bwd(logit_new, action, lse, dlp, g_out))


lm_policy_fwd.register_autograd(_lm_policy_backward, setup_context=_lm_policy_setup)


@torch.library.custom_op('b200rl::token_head_fwd', mutates_args=())
def token_head_fwd(lp_new: Tensor, lp_old: Tensor, lp_ref: Optional[Tensor], adv: Optional[Tensor],
                   reward: Optional[Tensor], weight: Optional[Tensor], clip_ratio: float,
                   beta: float) -> tuple[Tensor, Tensor]:
    """the GRPO (``lp_ref`` given) or RLOO head on a custom log_prob_fn's (B, S) fp32 output -> (loss / approx_kl /
    clipfrac, d loss / d lp_new for a unit upstream gradient)"""
    return ops.token_head_fwd_(lp_new, lp_old, lp_ref, adv, reward, weight, clip_ratio, beta)


@token_head_fwd.register_fake
def _(lp_new, lp_old, lp_ref, adv, reward, weight, clip_ratio, beta):
    return _f32(lp_new, 3), torch.empty_like(lp_new)


def _token_head_setup(ctx, inputs, output):
    ctx.save_for_backward(output[1])
    ctx.mark_non_differentiable(output[1])


def _token_head_backward(ctx, g_out, _g_dlp):
    dlp, = ctx.saved_tensors
    return _input_grads(token_head_fwd, lp_new=scale(g_out[:1], dlp))


token_head_fwd.register_autograd(_token_head_backward, setup_context=_token_head_setup)


@torch.library.custom_op('b200rl::ppo_lm_fwd', mutates_args=())
def ppo_lm_fwd(logit_new: Tensor, logit_old: Tensor, logit_pre: Optional[Tensor], action: Tensor, adv: Tensor,
               weight: Optional[Tensor], clip_ratio: float, dual_clip: float, kl_type: int,
               entropy: bool) -> tuple[Tensor, Tensor, Tensor, Tensor, Tensor]:
    """ppo_policy_error on token rows -> (policy / entropy / kl / approx_kl / clipfrac, and per row: logsumexp, entropy
    (empty without ``entropy``), the policy term's unit coefficient, the kl term's (empty without logit_pre))"""
    xs = [ops.logits_c(x) if x is not None else None for x in (logit_new, logit_old, logit_pre)]
    out, lse, ent, dpol, dkl = ops.ppo_lm_fwd_(xs[0], xs[1], xs[2], action, adv, weight, ops.logit_dtype(xs[0]),
                                               clip_ratio, dual_clip, kl_type, entropy, None, None, None)
    return out, lse, ent if ent is not None else _empty(out), dpol, dkl if dkl is not None else _empty(out)


@ppo_lm_fwd.register_fake
def _(logit_new, logit_old, logit_pre, action, adv, weight, clip_ratio, dual_clip, kl_type, entropy):
    rows = _rows(logit_new)
    return (_f32(logit_new, 5), _f32(logit_new, rows), _f32(logit_new, rows if entropy else 0), _f32(logit_new, rows),
            _f32(logit_new, rows if logit_pre is not None else 0))


@torch.library.custom_op('b200rl::ppo_lm_bwd', mutates_args=())
def ppo_lm_bwd(logit_new: Tensor, action: Tensor, weight: Optional[Tensor], lse: Tensor, ent: Tensor, dpol: Tensor,
               dkl: Tensor, g_out: Tensor) -> Tensor:
    """-> d / d logit_new for the upstream gradients g_out[0:3] of policy, entropy and kl loss"""
    x = ops.logits_c(logit_new)
    keep, upstream = _upstream(g_out, 3)
    return ops.ppo_lm_bwd_(ops.logit_dtype(x), x, action, weight, lse, ent if ent.numel() else None, dpol,
                           dkl if dkl.numel() else None, upstream, None, None, torch.empty_like(logit_new))


@ppo_lm_bwd.register_fake
def _(logit_new, *args):
    return torch.empty_like(logit_new)


def _ppo_lm_setup(ctx, inputs, output):
    a = _bind(ppo_lm_fwd, inputs)
    ctx.save_for_backward(a.logit_new, a.action, a.weight, *output[1:])
    ctx.set_materialize_grads(False)
    ctx.mark_non_differentiable(*output[1:])


def _ppo_lm_backward(ctx, g_out, *_):
    if g_out is None:
        return _input_grads(ppo_lm_fwd)
    return _input_grads(ppo_lm_fwd, logit_new=ppo_lm_bwd(*ctx.saved_tensors, g_out))


ppo_lm_fwd.register_autograd(_ppo_lm_backward, setup_context=_ppo_lm_setup)


@torch.library.custom_op('b200rl::a2c_lm_fwd', mutates_args=())
def a2c_lm_fwd(logit: Tensor, value: Tensor, action: Tensor, adv: Tensor, return_: Tensor,
               weight: Optional[Tensor]) -> tuple[Tensor, Tensor]:
    """a2c_error on token rows, value fp32 -> (policy / value / entropy loss, (4, rows): per row logsumexp, entropy, the
    policy term's unit coefficient, d value_loss / d value)"""
    x = ops.logits_c(logit)
    return ops.a2c_lm_fwd_(x, value, action, adv, return_, weight, ops.logit_dtype(x), None, None, None, None)


@a2c_lm_fwd.register_fake
def _(logit, value, action, adv, return_, weight):
    return _f32(logit, 3), _f32(logit, (4, _rows(logit)))


@torch.library.custom_op('b200rl::a2c_lm_bwd', mutates_args=())
def a2c_lm_bwd(logit: Tensor, value: Tensor, action: Tensor, weight: Optional[Tensor], per_row: Tensor,
               g_out: Tensor) -> tuple[Tensor, Tensor]:
    """-> (d / d logit, d / d value) for the upstream gradients g_out[0:3] of policy, value and entropy loss"""
    x = ops.logits_c(logit)
    keep, upstream = _upstream(g_out, 3)
    return ops.a2c_lm_bwd_(ops.logit_dtype(x), x, action, weight, *per_row.unbind(0), upstream, None, None,
                           torch.empty_like(logit), torch.empty_like(value))


@a2c_lm_bwd.register_fake
def _(logit, value, *args):
    return torch.empty_like(logit), torch.empty_like(value)


def _a2c_lm_setup(ctx, inputs, output):
    a = _bind(a2c_lm_fwd, inputs)
    ctx.save_for_backward(a.logit, a.value, a.action, a.weight, output[1])
    ctx.set_materialize_grads(False)
    ctx.mark_non_differentiable(output[1])


def _a2c_lm_backward(ctx, g_out, _g_per_row):
    if g_out is None:
        return _input_grads(a2c_lm_fwd)
    grad_logit, grad_value = a2c_lm_bwd(*ctx.saved_tensors, g_out)
    return _input_grads(a2c_lm_fwd, logit=grad_logit, value=grad_value)


a2c_lm_fwd.register_autograd(_a2c_lm_backward, setup_context=_a2c_lm_setup)


# ---------------------------------------------------------------------------------------------------------------------
# The language-model losses from the lm_head's hidden states (rl_utils/lm_linear.py): the op's body is eager's whole chunk
# loop (ops.lm_chunks_: logit GEMM, in-place row launch, dH / dW GEMMs), so the compiler sees one opaque op per call.  Here
# the GEMMs are the cost, so the gradient is not recomputed: as in eager mode the forward op writes dH / dW (and A2C's
# d value) for a unit upstream gradient, each only when ``want_*`` says so, and the backward op scales them out of place
# (b200rl_lm_linear_scale_out, the bits of eager's in-place scale; A2C's fp32 d value through ``scale``).  A repeated
# backward rescales the same saved unit gradients.  Not wanted, a gradient output is an empty tensor.
# ---------------------------------------------------------------------------------------------------------------------
def _or_empty(x, like):
    return x if x is not None else _empty(like)


@torch.library.custom_op('b200rl::lm_linear_loss', mutates_args=())
def lm_linear_loss_op(hidden: Tensor, lm_weight: Tensor, action: Tensor, lp_old: Tensor, lp_ref: Optional[Tensor],
                   side: Tensor, weight: Optional[Tensor], kind: str, B: int, S: int, dt: int, clip_ratio: float,
                   beta: float, want_dh: bool, want_dw: bool) -> tuple[Tensor, Tensor, Tensor]:
    """grpo / rloo_policy_error_linear on hidden (N, D), lm_weight (V, D) -> (loss / approx_kl / clipfrac, dH, dW)"""
    out, dh, dw = ops.lm_linear_loss_(hidden, lm_weight, action, lp_old, lp_ref, side, weight, kind, B, S, dt, clip_ratio,
                                      beta, want_dh, want_dw)
    return out, _or_empty(dh, hidden), _or_empty(dw, lm_weight)


@lm_linear_loss_op.register_fake
def _(hidden, lm_weight, action, lp_old, lp_ref, side, weight, kind, B, S, dt, clip_ratio, beta, want_dh, want_dw):
    return (_f32(hidden, 3), torch.empty_like(hidden) if want_dh else _empty(hidden),
            torch.empty_like(lm_weight) if want_dw else _empty(lm_weight))


@torch.library.custom_op('b200rl::lm_linear_pg', mutates_args=())
def lm_linear_pg_op(hidden: Tensor, lm_weight: Tensor, value: Optional[Tensor], action: Tensor, adv: Tensor,
                 weight: Optional[Tensor], lp_old: Optional[Tensor], lp_pre: Optional[Tensor], ret: Optional[Tensor],
                 kind: str, dt: int, clip_ratio: float, dual_clip: float, kl_type: int, entropy: bool, w_ent: float,
                 w_kl: float, w_val: float, want_dh: bool, want_dw: bool,
                 want_dv: bool) -> tuple[Tensor, Tensor, Tensor, Tensor, Tensor]:
    """ppo_policy_error_linear / a2c_error_linear -> (the one loss, the raw sums (PPO 5, A2C 3), dH, dW, d value (N)
    fp32); the loss is eager's ``ops.lm_pg_loss_`` of the sums"""
    cfg = (clip_ratio, dual_clip, kl_type, entropy, w_ent, w_kl, w_val)
    out, dh, dw, dv = ops.lm_linear_pg_(hidden, lm_weight, action, adv, weight, lp_old, lp_pre, value, ret, kind, dt, cfg,
                                        want_dh, want_dw, want_dv)
    return ops.lm_pg_loss_(out, kind, cfg), out, _or_empty(dh, hidden), _or_empty(dw, lm_weight), _or_empty(dv, out)


@lm_linear_pg_op.register_fake
def _(hidden, lm_weight, value, action, adv, weight, lp_old, lp_pre, ret, kind, dt, clip_ratio, dual_clip, kl_type,
      entropy, w_ent, w_kl, w_val, want_dh, want_dw, want_dv):
    return (_f32(hidden, ()), _f32(hidden, 5 if kind == 'ppo' else 3),
            torch.empty_like(hidden) if want_dh else _empty(hidden),
            torch.empty_like(lm_weight) if want_dw else _empty(lm_weight), _f32(hidden, hidden.shape[0] if want_dv else 0))


@torch.library.custom_op('b200rl::lm_linear_scale_out', mutates_args=())
def lm_linear_scale_out(g: Tensor, x: Tensor) -> Tensor:
    """``g * x`` into a fresh contiguous tensor of x's shape and dtype (fp32 or bf16, any layout) for a one-element
    upstream gradient ``g``"""
    kg, pg = _one(g)
    return ops.lm_scale_out_(ops.logit_dtype(x), pg, x)


@lm_linear_scale_out.register_fake
def _(g, x):
    return x.new_empty(x.shape)


def _lm_linear_loss_setup(ctx, inputs, output):
    a = _bind(lm_linear_loss_op, inputs)
    ctx.save_for_backward(output[1], output[2])
    ctx.want = (a.want_dh, a.want_dw)
    ctx.set_materialize_grads(False)
    ctx.mark_non_differentiable(output[1], output[2])


def _lm_linear_loss_backward(ctx, g_out, _g_dh, _g_dw):
    if g_out is None:
        return _input_grads(lm_linear_loss_op)
    dh, dw = ctx.saved_tensors
    want_dh, want_dw = ctx.want
    g = g_out[:1]  # the loss's; approx_kl and clipfrac leave the wrapper detached
    return _input_grads(lm_linear_loss_op, hidden=lm_linear_scale_out(g, dh) if want_dh else None,
                        lm_weight=lm_linear_scale_out(g, dw) if want_dw else None)


lm_linear_loss_op.register_autograd(_lm_linear_loss_backward, setup_context=_lm_linear_loss_setup)


def _lm_linear_pg_setup(ctx, inputs, output):
    a = _bind(lm_linear_pg_op, inputs)
    ctx.save_for_backward(*output[2:])
    ctx.want = (a.want_dh, a.want_dw, a.want_dv)
    ctx.set_materialize_grads(False)
    ctx.mark_non_differentiable(*output[1:])


def _lm_linear_pg_backward(ctx, g_loss, *_):
    if g_loss is None:
        return _input_grads(lm_linear_pg_op)
    dh, dw, dv = ctx.saved_tensors
    want_dh, want_dw, want_dv = ctx.want
    return _input_grads(lm_linear_pg_op, hidden=lm_linear_scale_out(g_loss, dh) if want_dh else None,
                        lm_weight=lm_linear_scale_out(g_loss, dw) if want_dw else None,
                        value=scale(g_loss, dv) if want_dv else None)


lm_linear_pg_op.register_autograd(_lm_linear_pg_backward, setup_context=_lm_linear_pg_setup)


@torch.library.custom_op('b200rl::lm_logp', mutates_args=())
def lm_logp_op(hidden: Tensor, lm_weight: Tensor, index: Tensor, dt: int) -> tuple[Tensor, Tensor]:
    """token_logp_linear -> (log p(index), logsumexp), fp32 per token row"""
    return ops.lm_logp_fwd_(hidden, lm_weight, index, dt)


@lm_logp_op.register_fake
def _(hidden, lm_weight, index, dt):
    return _f32(hidden, hidden.shape[0]), _f32(hidden, hidden.shape[0])


@torch.library.custom_op('b200rl::lm_logp_bwd', mutates_args=())
def lm_logp_bwd(hidden: Tensor, lm_weight: Tensor, index: Tensor, lse: Tensor, g: Tensor, dt: int, want_dh: bool,
                want_dw: bool) -> tuple[Tensor, Tensor]:
    """-> (dH, dW) for the upstream gradient g (N) of log p: per chunk the logit GEMM again, as in eager mode"""
    dh, dw = ops.lm_logp_bwd_(hidden, lm_weight, index, lse, g.float().contiguous(), dt, want_dh, want_dw)
    return _or_empty(dh, hidden), _or_empty(dw, lm_weight)


@lm_logp_bwd.register_fake
def _(hidden, lm_weight, index, lse, g, dt, want_dh, want_dw):
    return (torch.empty_like(hidden) if want_dh else _empty(hidden),
            torch.empty_like(lm_weight) if want_dw else _empty(lm_weight))


def _lm_logp_setup(ctx, inputs, output):
    a = _bind(lm_logp_op, inputs)
    ctx.save_for_backward(a.hidden, a.lm_weight, a.index, output[1])
    ctx.dt = a.dt
    ctx.mark_non_differentiable(output[1])


def _lm_logp_backward(ctx, g, _g_lse):
    hidden, lm_weight, index, lse = ctx.saved_tensors
    want_dh, want_dw = ctx.needs_input_grad[:2]
    dh, dw = lm_logp_bwd(hidden, lm_weight, index, lse, g, ctx.dt, want_dh, want_dw)
    return _input_grads(lm_logp_op, hidden=dh if want_dh else None, lm_weight=dw if want_dw else None)


lm_logp_op.register_autograd(_lm_logp_backward, setup_context=_lm_logp_setup)


# ---------------------------------------------------------------------------------------------------------------------
# the advantage statistics of PPOPolicy / PPOFPolicy (csrc/policy.cu): no gradient, as in the reference
# ---------------------------------------------------------------------------------------------------------------------
@torch.library.custom_op('b200rl::gae_returns', mutates_args=())
def gae_returns_op(value: Tensor, next_value: Tensor, reward: Tensor, done: Optional[Tensor], traj_flag: Optional[Tensor],
                   gamma: float, lambda_: float, vscale: float) -> tuple[Tensor, Tensor, Tensor, Tensor, Tensor, Tensor]:
    """gae_returns -> (adv, unnormalized return, value_out, return_out, return_stats, adv_stats); value_out / return_out
    are empty when ``vscale`` is 0 (no value_norm).  The inputs are not modified."""
    adv, unnorm, vout, rout, stats, astats = ops.gae_returns_(value, next_value, reward, done, traj_flag, gamma, lambda_, 1,
                                                              vscale, True, True, want_adv_stats=True)
    return (adv, unnorm, vout if vout is not None else _empty(adv), rout if rout is not None else _empty(adv), stats,
            astats)


@gae_returns_op.register_fake
def _(value, next_value, reward, done, traj_flag, gamma, lambda_, vscale):
    scaled = (lambda: torch.empty_like(value)) if vscale != 0.0 else (lambda: _empty(value))
    return (torch.empty_like(value), torch.empty_like(value), scaled(), scaled(), _f32(value, 3), _f32(value, 2))


@torch.library.custom_op('b200rl::gae_returns_norm', mutates_args=())
def gae_returns_norm(value: Tensor, next_value: Tensor, reward: Tensor, done: Optional[Tensor],
                     traj_flag: Optional[Tensor], gamma: float, lambda_: float, value_norm: str, std: float,
                     mu: Optional[Tensor], sigma: Optional[Tensor]) -> tuple[Tensor, Tensor, Tensor, Tensor, Tensor]:
    """ppof_gae_returns -> (adv, value_out, return_out, return_stats (empty unless 'baseline'), adv_stats)"""
    adv, vout, rout, stats, astats = ops.gae_returns_norm_(value, next_value, reward, done, traj_flag, gamma, lambda_,
                                                           value_norm, std, mu, sigma, value_norm == 'baseline')
    return adv, vout, rout, stats if stats is not None else _empty(adv), astats


@gae_returns_norm.register_fake
def _(value, next_value, reward, done, traj_flag, gamma, lambda_, value_norm, std, mu, sigma):
    return (torch.empty_like(value), torch.empty_like(value), torch.empty_like(value),
            _f32(value, 3 if value_norm == 'baseline' else 0), _f32(value, 2))


@torch.library.custom_op('b200rl::adv_stats', mutates_args=())
def adv_stats_op(x: Tensor) -> Tensor:
    """{mean, std (unbiased) + 1e-8} of ``x``"""
    return ops.adv_stats_(x)


@adv_stats_op.register_fake
def _(x):
    return _f32(x, 2)


@torch.library.custom_op('b200rl::normalize', mutates_args=())
def normalize_op(x: Tensor, stats: Tensor) -> Tensor:
    return ops.normalize_(x, stats)


@normalize_op.register_fake
def _(x, stats):
    return torch.empty_like(x)


# ---------------------------------------------------------------------------------------------------------------------
# symlog / inv_symlog
# ---------------------------------------------------------------------------------------------------------------------
@torch.library.custom_op('b200rl::value_map', mutates_args=())
def value_map_op(x: Tensor, mode: int) -> Tensor:
    """symlog (``mode`` 0) or inv_symlog (1) of a contiguous fp32 tensor"""
    return ops.value_map_fwd_(x, mode)


@value_map_op.register_fake
def _(x, mode):
    return torch.empty_like(x)


@torch.library.custom_op('b200rl::value_map_bwd', mutates_args=())
def value_map_bwd(x: Tensor, g: Tensor, mode: int) -> Tensor:
    return ops.value_map_bwd_(x, ops.f32c(g, 'grad'), mode)


@value_map_bwd.register_fake
def _(x, g, mode):
    return torch.empty_like(x)


def _value_map_setup(ctx, inputs, output):
    a = _bind(value_map_op, inputs)
    ctx.save_for_backward(a.x)
    ctx.mode = a.mode


def _value_map_backward(ctx, g):
    x, = ctx.saved_tensors
    return _input_grads(value_map_op, x=value_map_bwd(x, g, ctx.mode))


value_map_op.register_autograd(_value_map_backward, setup_context=_value_map_setup)


# ---------------------------------------------------------------------------------------------------------------------
# qrdqn / iqn / fqf_nstep_td_error: the op reads the element strides of (sample, quantile[, action]) from its tensors
# ---------------------------------------------------------------------------------------------------------------------
QUANTILE_AXES = ((0, 2, 1), (1, 0, 2), (0, 1, 2))  # the (sample, quantile, action) axes of q per form: QR-DQN, IQN, FQF


def _quantile_strides(t, form):
    return tuple(t.stride(a) for a in QUANTILE_AXES[form])


@torch.library.custom_op('b200rl::quantile_fwd', mutates_args=())
def quantile_fwd(q: Tensor, next_n_q: Tensor, action: Tensor, next_n_action: Tensor, reward: Tensor, done: Tensor,
                 tau: Tensor, weight: Optional[Tensor], value_gamma: Optional[Tensor], value_gamma_scalar: Optional[float],
                 vg_stride: int, B: int, N: int, n_tau: int, n_tau_prime: int, nstep: int, gamma: float, form: int,
                 kappa: float, want_grad: bool) -> tuple[Tensor, Tensor, Tensor, Tensor]:
    """-> (loss, td, dtheta, grad_unit); grad_unit is empty without ``want_grad``.  ``tau`` (B, n_tau) may be any strided
    view, as in eager mode."""
    if value_gamma_scalar is not None:
        value_gamma = ops.const_scalar(value_gamma_scalar, q.device)
    loss, td, dtheta, grad_unit = ops.quantile_fwd_(
        q, next_n_q, action, next_n_action, reward, done, tau, weight, value_gamma, vg_stride, B, N, n_tau, n_tau_prime,
        nstep, gamma, _quantile_strides(q, form), _quantile_strides(next_n_q, form), (tau.stride(0), tau.stride(1)), form,
        kappa, want_grad)
    return loss, td, dtheta, grad_unit if grad_unit is not None else _empty(loss)


@quantile_fwd.register_fake
def _(q, next_n_q, action, next_n_action, reward, done, tau, weight, value_gamma, value_gamma_scalar, vg_stride, B, N,
      n_tau, n_tau_prime, nstep, gamma, form, kappa, want_grad):
    loss = q.new_empty(())
    return loss, q.new_empty(B), q.new_empty(B, n_tau), torch.empty_like(q) if want_grad else _empty(loss)


@torch.library.custom_op('b200rl::quantile_bwd', mutates_args=())
def quantile_bwd(dtheta: Tensor, weight: Optional[Tensor], action: Tensor, g_loss: Optional[Tensor],
                 g_td: Optional[Tensor], grad_unit: Tensor, B: int, N: int, n_tau: int, form: int) -> Tensor:
    """-> d / d q; verifies a copy of the forward-written unit gradient when only the loss has a gradient"""
    kl, pg = _one(g_loss)
    kt, ptd = _one(g_td)
    # the forward writes grad_unit whenever q wants a gradient, so it is never empty here; a fresh buffer takes its
    # strides, which the launch reads
    grad, skip = _unit_grad(grad_unit, (g_td, ), lambda: torch.empty_like(grad_unit))
    return ops.quantile_bwd_(dtheta, weight, action, pg, ptd, B, N, n_tau, _quantile_strides(grad, form), skip, grad)


@quantile_bwd.register_fake
def _(dtheta, weight, action, g_loss, g_td, grad_unit, B, N, n_tau, form):
    return torch.empty_like(grad_unit)


def _quantile_setup(ctx, inputs, output):
    a = _bind(quantile_fwd, inputs)
    ctx.save_for_backward(output[2], a.weight, a.action, output[3])
    ctx.cfg = (a.B, a.N, a.n_tau, a.form)
    ctx.set_materialize_grads(False)
    ctx.mark_non_differentiable(*output[2:])


def _quantile_backward(ctx, g_loss, g_td, *_):
    if g_loss is None and g_td is None:
        return _input_grads(quantile_fwd)
    dtheta, weight, action, grad_unit = ctx.saved_tensors
    return _input_grads(quantile_fwd, q=quantile_bwd(dtheta, weight, action, g_loss, g_td, grad_unit, *ctx.cfg))


quantile_fwd.register_autograd(_quantile_backward, setup_context=_quantile_setup)


# ---------------------------------------------------------------------------------------------------------------------
# fqf_calculate_fraction_loss: the op reads the element strides of q_tau_i, q_value and quantiles from its tensors; the
# gradient goes to quantiles only
# ---------------------------------------------------------------------------------------------------------------------
@torch.library.custom_op('b200rl::fqf_fraction_fwd', mutates_args=())
def fqf_fraction_fwd(q_tau_i: Tensor, q_value: Tensor, quantiles: Tensor, action: Tensor, B: int, N: int,
                     want_grad: bool) -> tuple[Tensor, Tensor, Tensor]:
    """-> (loss, g (B, N-1), grad_unit (B, N+1)); grad_unit is empty without ``want_grad``.  q_tau_i (B, N-1, A'),
    q_value (B, N, A) and quantiles (B, N+1) may be any strided views, as in eager mode."""
    loss, g, grad_unit = ops.fqf_fraction_fwd_(q_tau_i, q_value, quantiles, action, B, N, q_tau_i.stride(),
                                               q_value.stride(), quantiles.stride(), want_grad)
    return loss, g, grad_unit if grad_unit is not None else _empty(loss)


@fqf_fraction_fwd.register_fake
def _(q_tau_i, q_value, quantiles, action, B, N, want_grad):
    loss = quantiles.new_empty(())
    return loss, quantiles.new_empty(B, N - 1), quantiles.new_empty(B, N + 1) if want_grad else _empty(loss)


@torch.library.custom_op('b200rl::fqf_fraction_bwd', mutates_args=())
def fqf_fraction_bwd(g: Tensor, g_loss: Tensor, grad_unit: Tensor, B: int, N: int) -> Tensor:
    """-> d / d quantiles (B, N+1); verifies a copy of the forward-written unit gradient when there is one"""
    kl, pg = _one(g_loss)
    grad, skip = _unit_grad(grad_unit, (), lambda: g.new_empty(B, N + 1))  # g, the other output, is not differentiable
    return ops.fqf_fraction_bwd_(g, pg, B, N, skip, grad)


@fqf_fraction_bwd.register_fake
def _(g, g_loss, grad_unit, B, N):
    return g.new_empty(B, N + 1)


def _fqf_fraction_setup(ctx, inputs, output):
    a = _bind(fqf_fraction_fwd, inputs)
    ctx.save_for_backward(output[1], output[2])
    ctx.cfg = (a.B, a.N)
    ctx.set_materialize_grads(False)
    ctx.mark_non_differentiable(*output[1:])


def _fqf_fraction_backward(ctx, g_loss, *_):
    if g_loss is None:
        return _input_grads(fqf_fraction_fwd)
    g, grad_unit = ctx.saved_tensors
    return _input_grads(fqf_fraction_fwd, quantiles=fqf_fraction_bwd(g, g_loss, grad_unit, *ctx.cfg))


fqf_fraction_fwd.register_autograd(_fqf_fraction_backward, setup_context=_fqf_fraction_setup)


# ---------------------------------------------------------------------------------------------------------------------
# ppo_error_continuous and its policy-only / HAPPO call sites (csrc/heads.cu): the forward launch always writes the
# gradients for the call site's record when a gradient is wanted, so the backward op always verifies a copy
# ---------------------------------------------------------------------------------------------------------------------
@torch.library.custom_op('b200rl::ppoc_loss', mutates_args=())
def ppoc_loss(mu: Tensor, sigma: Tensor, value_new: Tensor, mu_old: Tensor, sigma_old: Tensor, mu_pre: Optional[Tensor],
              sigma_pre: Optional[Tensor], action: Tensor, value_old: Tensor, adv: Tensor, return_: Tensor,
              weight: Optional[Tensor], factor: Optional[Tensor], S: int, D: int, clip_ratio: float, use_value_clip: int,
              dual_clip: float, kl_type: int, hint_kind: str,
              want_grad: bool) -> tuple[Tensor, Tensor, Tensor, Tensor, Tensor]:
    """-> (the six floats the launch writes: policy, value, entropy, kl loss, approx_kl, clipfrac; grad_mu, grad_sigma,
    grad_value, g_used); the last four are empty without ``want_grad``"""
    saved = (mu, sigma, value_new, mu_old, sigma_old, mu_pre, sigma_pre, action, value_old, adv, return_, weight)
    out, spec = ops.ppoc_fwd_(saved, (factor, S, D, clip_ratio, use_value_clip, dual_clip, kl_type), hint_kind, want_grad)
    out = out[:6]
    if not want_grad:
        return (out, ) + (_empty(out), ) * 4
    return (out, ) + spec


@ppoc_loss.register_fake
def _(mu, sigma, value_new, mu_old, sigma_old, mu_pre, sigma_pre, action, value_old, adv, return_, weight, factor, S, D,
      clip_ratio, use_value_clip, dual_clip, kl_type, hint_kind, want_grad):
    out = mu.new_empty(6)
    if not want_grad:
        return (out, ) + (_empty(out), ) * 4
    return out, torch.empty_like(mu), torch.empty_like(sigma), torch.empty_like(value_new), out.new_empty(4)


@torch.library.custom_op('b200rl::ppoc_bwd', mutates_args=())
def ppoc_bwd(mu: Tensor, sigma: Tensor, value_new: Tensor, mu_old: Tensor, sigma_old: Tensor, mu_pre: Optional[Tensor],
             sigma_pre: Optional[Tensor], action: Tensor, value_old: Tensor, adv: Tensor, return_: Tensor,
             weight: Optional[Tensor], factor: Optional[Tensor], g_out: Tensor, grad_mu: Tensor, grad_sigma: Tensor,
             grad_value: Tensor, g_used: Tensor, S: int, D: int, clip_ratio: float, use_value_clip: int, dual_clip: float,
             kl_type: int, hint_kind: str) -> tuple[Tensor, Tensor, Tensor]:
    """-> (grad_mu, grad_sigma, grad_value) for the upstream gradients g_out[0:4] of policy, value, entropy and kl loss"""
    keep, upstream = _upstream(g_out, 4)
    saved = (mu, sigma, value_new, mu_old, sigma_old, mu_pre, sigma_pre, action, value_old, adv, return_, weight)
    cfg = (factor, S, D, clip_ratio, use_value_clip, dual_clip, kl_type)
    return ops.ppoc_bwd_(saved, cfg, upstream, _forward_grads(True, g_used, grad_mu, grad_sigma, grad_value), hint_kind)


@ppoc_bwd.register_fake
def _(mu, sigma, value_new, *args):
    return torch.empty_like(mu), torch.empty_like(sigma), torch.empty_like(value_new)


def _ppoc_setup(ctx, inputs, output):
    a = _bind(ppoc_loss, inputs)
    ctx.save_for_backward(a.mu, a.sigma, a.value_new, a.mu_old, a.sigma_old, a.mu_pre, a.sigma_pre, a.action, a.value_old,
                          a.adv, a.return_, a.weight, a.factor, *output[1:])
    ctx.cfg = (a.S, a.D, a.clip_ratio, a.use_value_clip, a.dual_clip, a.kl_type, a.hint_kind)
    ctx.set_materialize_grads(False)
    ctx.mark_non_differentiable(*output[1:])


def _ppoc_backward(ctx, g_out, *_):
    if g_out is None:
        return _input_grads(ppoc_loss)
    saved = ctx.saved_tensors
    grad_mu, grad_sigma, grad_value = ppoc_bwd(*saved[:13], g_out, *saved[13:], *ctx.cfg)
    return _input_grads(ppoc_loss, mu=grad_mu, sigma=grad_sigma, value_new=grad_value)


ppoc_loss.register_autograd(_ppoc_backward, setup_context=_ppoc_setup)


# ---------------------------------------------------------------------------------------------------------------------
# coma_error (csrc/td.cu HEAD 2 + csrc/pg.cu): as ppoc, the forward launch writes the gradients for the 'coma' record
# whenever a gradient is wanted, so the backward op always verifies a copy.  The differentiable-returns path (target_q_value
# or reward requiring grad) is not traced: it runs generalized_lambda_returns' autograd function, as in eager mode
# ---------------------------------------------------------------------------------------------------------------------
@torch.library.custom_op('b200rl::coma_fwd', mutates_args=())
def coma_fwd(logit: Tensor, q_value: Tensor, target_q: Tensor, action: Tensor, reward: Tensor, weight: Optional[Tensor],
             T: int, B: int, A: int, N: int, gamma: float, lambda_: float,
             want_grad: bool) -> tuple[Tensor, Tensor, Tensor, Tensor, Tensor, Tensor]:
    """-> (policy / value / entropy loss, adv, dq, grad_logit, grad_q_value, g_used); the last three are empty without
    ``want_grad``"""
    out, adv, dq, _, spec = ops.coma_fwd_(logit, q_value, target_q, action, reward, weight, T, B, A, N, gamma, lambda_,
                                          want_grad, False)
    if not want_grad:
        return (out, adv, dq) + (_empty(out), ) * 3
    return (out, adv, dq) + spec


@coma_fwd.register_fake
def _(logit, q_value, target_q, action, reward, weight, T, B, A, N, gamma, lambda_, want_grad):
    out = logit.new_empty(3)
    adv, dq = logit.new_empty(T * B * A), logit.new_empty((T - 1) * B * A)
    if not want_grad:
        return (out, adv, dq) + (_empty(out), ) * 3
    return out, adv, dq, torch.empty_like(logit), torch.empty_like(q_value), out.new_empty(4)


@torch.library.custom_op('b200rl::coma_bwd', mutates_args=())
def coma_bwd(logit: Tensor, action: Tensor, weight: Optional[Tensor], adv: Tensor, dq: Tensor, g_out: Tensor,
             grad_logit: Tensor, grad_q: Tensor, g_used: Tensor, T: int, B: int, A: int, N: int) -> tuple[Tensor, Tensor]:
    """-> (grad_logit, grad_q_value) for the upstream gradients g_out[0:3] of policy, value and entropy loss"""
    keep, upstream = _upstream(g_out, 3)
    spec = _forward_grads(True, g_used, grad_logit, grad_q)
    return ops.coma_bwd_(logit, action, weight, adv, dq, T, B, A, N, upstream, spec)


@coma_bwd.register_fake
def _(logit, action, weight, adv, dq, g_out, grad_logit, grad_q, *args):
    return torch.empty_like(logit), torch.empty_like(grad_q)


def _coma_setup(ctx, inputs, output):
    a = _bind(coma_fwd, inputs)
    ctx.save_for_backward(a.logit, a.action, a.weight, *output[1:])
    ctx.cfg = (a.T, a.B, a.A, a.N)
    ctx.set_materialize_grads(False)
    ctx.mark_non_differentiable(*output[1:])


def _coma_backward(ctx, g_out, *_):
    if g_out is None:
        return _input_grads(coma_fwd)
    grad_logit, grad_q = coma_bwd(*ctx.saved_tensors[:5], g_out, *ctx.saved_tensors[5:], *ctx.cfg)
    return _input_grads(coma_fwd, logit=grad_logit, q_value=grad_q)


coma_fwd.register_autograd(_coma_backward, setup_context=_coma_setup)


# ---------------------------------------------------------------------------------------------------------------------
# ScatterConnection (csrc/scatter.cu): x and the index operands keep their strides
# ---------------------------------------------------------------------------------------------------------------------
@torch.library.custom_op('b200rl::scatter_fwd', mutates_args=())
def scatter_fwd(x: Tensor, row: Tensor, col: Tensor, H: int, W: int, mode: int) -> Tensor:
    return ops.scatter_fwd_(x, row, col, H, W, mode)


@scatter_fwd.register_fake
def _(x, row, col, H, W, mode):
    return x.new_empty(x.shape[0], x.shape[2], H, W)


@torch.library.custom_op('b200rl::scatter_bwd', mutates_args=())
def scatter_bwd(g: Tensor, row: Tensor, col: Tensor, M: int, H: int, W: int) -> Tensor:
    return ops.scatter_bwd_(g, row, col, M, H, W)


@scatter_bwd.register_fake
def _(g, row, col, M, H, W):
    return g.new_empty(g.shape[0], M, g.shape[1], dtype=torch.float32)


def _scatter_setup(ctx, inputs, output):
    a = _bind(scatter_fwd, inputs)
    ctx.save_for_backward(a.row, a.col)
    ctx.cfg = (a.x.shape[1], a.H, a.W)


def _scatter_backward(ctx, g):
    row, col = ctx.saved_tensors
    return _input_grads(scatter_fwd, x=scatter_bwd(g, row, col, *ctx.cfg))


scatter_fwd.register_autograd(_scatter_backward, setup_context=_scatter_setup)


# ---------------------------------------------------------------------------------------------------------------------
# The layer-normalised LSTM (csrc/lstm.cu, GEMMs on cuBLAS): one op per layer per call in each direction
# ---------------------------------------------------------------------------------------------------------------------
@torch.library.custom_op('b200rl::lnlstm_fwd', mutates_args=())
def lnlstm_fwd(x: Tensor, h0: Tensor, c0: Tensor, wx: Tensor, wh: Tensor, bias: Tensor, gamma_x: Tensor, beta_x: Tensor,
               gamma_h: Tensor, beta_h: Tensor,
               save: bool) -> tuple[Tensor, Tensor, Tensor, Tensor, Tensor, Tensor, Tensor]:
    """-> (y, h_T, c_T, GX, GH, C, stats), as ``ops.lnlstm_fwd_``"""
    out = ops.lnlstm_fwd_(x, h0, c0, wx, wh, bias, gamma_x, beta_x, gamma_h, beta_h, save)
    # a custom op returns tensors only, none aliasing another: stats is empty and C a copy of c_T where the eager path
    # keeps no statistics and shares c_T's memory
    C = out[5] if out[5].data_ptr() != out[2].data_ptr() else out[2].clone().view(out[5].shape)
    return out[:5] + (C, out[6] if out[6] is not None else x.new_empty(0))


@lnlstm_fwd.register_fake
def _(x, h0, c0, wx, wh, bias, gamma_x, beta_x, gamma_h, beta_h, save):
    T, B, _ = x.shape
    H = wh.shape[0]
    stats = x.new_empty(T, B, 4) if save else x.new_empty(0)
    return (x.new_empty(T, B, H), x.new_empty(B, H), x.new_empty(B, H), x.new_empty(T, B, 4 * H),
            x.new_empty(T if save else 1, B, 4 * H), x.new_empty(T, B, H), stats)


@torch.library.custom_op('b200rl::lnlstm_bwd', mutates_args=())
def lnlstm_bwd(g_y: Optional[Tensor], g_hT: Optional[Tensor], g_cT: Optional[Tensor], x: Tensor, h0: Tensor, c0: Tensor,
               wx: Tensor, wh: Tensor, bias: Tensor, gamma_x: Tensor, beta_x: Tensor, gamma_h: Tensor, beta_h: Tensor,
               y: Tensor, GX: Tensor, GH: Tensor, C: Tensor, stats: Tensor, needs: list[bool]) -> list[Tensor]:
    """-> the ten input gradients of ``lnlstm_fwd``; an input whose ``needs`` is false gets an empty tensor"""
    grads = ops.lnlstm_bwd_(g_y, g_hT, g_cT, x, h0, c0, wx, wh, bias, gamma_x, beta_x, gamma_h, beta_h, y, GX, GH, C,
                            stats, needs)
    return [x.new_empty(0) if g is None else g for g in grads]


@lnlstm_bwd.register_fake
def _(g_y, g_hT, g_cT, x, h0, c0, wx, wh, bias, gamma_x, beta_x, gamma_h, beta_h, y, GX, GH, C, stats, needs):
    ins = (x, h0, c0, wx, wh, bias, gamma_x, beta_x, gamma_h, beta_h)
    return [t.new_empty(t.shape) if n else x.new_empty(0) for t, n in zip(ins, needs)]  # contiguous, as the real op's


def _lnlstm_setup(ctx, inputs, output):
    a = _bind(lnlstm_fwd, inputs)
    ctx.save_for_backward(a.x, a.h0, a.c0, a.wx, a.wh, a.bias, a.gamma_x, a.beta_x, a.gamma_h, a.beta_h, *output[:1],
                          *output[3:])
    ctx.set_materialize_grads(False)
    ctx.mark_non_differentiable(*output[3:])


def _lnlstm_backward(ctx, g_y, g_hT, g_cT, *_):
    needs = list(ctx.needs_input_grad[:10])  # x ... beta_h: every argument but ``save``
    grads = lnlstm_bwd(g_y, g_hT, g_cT, *ctx.saved_tensors, needs)
    return _input_grads(lnlstm_fwd, **{n: g for n, g, need in zip(_names(lnlstm_fwd), grads, needs) if need})


lnlstm_fwd.register_autograd(_lnlstm_backward, setup_context=_lnlstm_setup)


# ---------------------------------------------------------------------------------------------------------------------
# The one entry point of each operator for rl_utils / torch_utils: the custom op above while torch.compile traces, and
# otherwise exactly eager mode's call -- the autograd.Function of ops, or its no-grad shortcut.  A python-scalar weight /
# value_gamma / is_expert comes in as a python number: eager mode reads it from a cached device constant, the custom ops
# take it as a float (they look the constant up when they run, so tracing allocates nothing).
# ---------------------------------------------------------------------------------------------------------------------
def _want_grad(*xs):
    return torch.is_grad_enabled() and any(x.requires_grad for x in xs)


def _is_scalar(x):
    return x is not None and not isinstance(x, Tensor)


def _scalar_or_tensor(x):
    """(tensor, None) or (None, python float): the custom ops take a python-scalar weight / value_gamma as a float"""
    return (None, float(x)) if _is_scalar(x) else (x, None)


def _const(x, dev):
    """eager mode's form of a python-scalar weight / value_gamma: the cached device constant"""
    return ops.const_scalar(x, dev) if _is_scalar(x) else x


def stage_logits(x):
    """language-model logits for the vocabulary-scale kernels: eager mode makes the 16-byte-aligned copy of an odd-offset
    view (ops.logits_c); a traced tensor has no address, so under compile the custom op makes that copy itself"""
    return x.contiguous() if torch.compiler.is_compiling() else ops.logits_c(x)


def gae(value, next_value, reward, done, traj_flag, gamma, lambda_, agents):
    """-> adv; next_value is masked in place by (1 - done)"""
    if not torch.compiler.is_compiling():
        return ops.gae_(value, next_value, reward, done, traj_flag, gamma, lambda_, agents)
    return gae_op(value, next_value, reward, done, traj_flag, float(gamma), float(lambda_), agents)


def ppo(logit_new, value_new, logit_old, action, value_old, adv, return_, weight, logit_pre, S, G, N, clip_ratio,
        use_value_clip, dual_clip, kl_type, hint_kind, adv_stats=None, factor=None):
    """-> (policy, value, entropy, kl loss, a vector whose [4:6] are approx_kl, clipfrac), as PPOFunction"""
    if not torch.compiler.is_compiling():
        return ops.PPOFunction.apply(logit_new, value_new, logit_old, action, value_old, adv, return_, weight, logit_pre,
                                     S, G, N, clip_ratio, use_value_clip, dual_clip, kl_type, hint_kind, adv_stats, factor)
    out = ppo_loss(logit_new, value_new, logit_old, action, value_old, adv, return_, weight, logit_pre, adv_stats, factor,
                   S, G, N, clip_ratio, use_value_clip, dual_clip, kl_type, hint_kind,
                   _want_grad(logit_new, value_new))[0]
    return out[0], out[1], out[2], out[3], out


def qntd(q, next_n_q, action, next_n_action, reward, done, weight, value_gamma, vg_stride, gamma_ps, S, G, N, nstep, gamma,
         cum_reward, rescale, eps, criterion, crit_param, group_mean):
    """-> (loss, td, target, priority; None under compile), as QNStepTDFunction without the sequence form"""
    if not torch.compiler.is_compiling():
        return ops.QNStepTDFunction.apply(q, next_n_q, action, next_n_action, reward, done, weight,
                                          _const(value_gamma, q.device), vg_stride, gamma_ps, S, G, N, nstep, gamma,
                                          cum_reward, rescale, eps, criterion, crit_param, group_mean, 0, 0.0, False)
    vg, vg_scalar = _scalar_or_tensor(value_gamma)
    loss, td, _, target, _ = qntd_fwd(q, next_n_q, action, next_n_action, reward, done, weight, vg, vg_scalar, vg_stride,
                                      gamma_ps, S, G, N, nstep, gamma, cum_reward, rescale, eps, criterion, crit_param,
                                      group_mean, _want_grad(q))
    return loss, td, target, None


def qntd_seq(q, next_n_q, action, next_n_action, reward, done, weight, value_gamma, vg_stride, gamma_ps, S, N, nstep, gamma,
             rescale, criterion, crit_param, seq_len, priority_mix):
    """-> (loss, td, priority), as QNStepTDFunction's sequence form"""
    if not torch.compiler.is_compiling():
        loss, td, _, prio = ops.QNStepTDFunction.apply(
            q, next_n_q, action, next_n_action, reward, done, weight, _const(value_gamma, q.device), vg_stride, gamma_ps,
            S, 1, N, nstep, gamma, 0, rescale, 1e-2, criterion, crit_param, 0, seq_len, priority_mix, True)
        return loss, td, prio
    vg, vg_scalar = _scalar_or_tensor(value_gamma)
    loss, td, _, prio, _ = qntd_seq_fwd(q, next_n_q, action, next_n_action, reward, done, weight, vg, vg_scalar, vg_stride,
                                        gamma_ps, S, N, nstep, gamma, rescale, criterion, crit_param, seq_len,
                                        priority_mix, _want_grad(q))
    return loss, td, prio


def dist_nstep_td(dist, next_n_dist, act, next_n_act, reward, done, weight, w_stride, value_gamma, vg_stride, B, A, N,
                  n_atom, nstep, gamma, v_min, v_max, check_positive):
    """-> (loss, td), as DistNStepTDFunction; with ``check_positive`` the reference's assertion that dist[b, act] > 0"""
    from .rl_utils.td import _support
    if not torch.compiler.is_compiling():
        dev = dist.device
        w, vg = _const(weight, dev), _const(value_gamma, dev)
        bad = torch.zeros(1, dtype=torch.int32, device=dev) if check_positive else None
        loss, td = ops.DistNStepTDFunction.apply(dist, next_n_dist, act, next_n_act, reward, done, w, w_stride, vg,
                                                 vg_stride, _support(v_min, v_max, n_atom, dev), B, A, N, n_atom, nstep,
                                                 gamma, v_min, v_max, bad)
        if check_positive:
            assert bad.item() == 0, ("dist act", "non-positive probability in dist[batch_range, act]")  # td.py:513
        return loss, td
    w, w_scalar = _scalar_or_tensor(weight)
    vg, vg_scalar = _scalar_or_tensor(value_gamma)
    loss, td, _, _ = dntd_fwd(dist, next_n_dist, act, next_n_act, reward, done, w, w_scalar, w_stride, vg, vg_scalar,
                              vg_stride, B, A, N, n_atom, nstep, gamma, v_min, v_max, check_positive, _want_grad(dist))
    return loss, td


def td_lambda(value, reward, weight, gamma, lambda_):
    if not torch.compiler.is_compiling():
        return ops.td_lambda_(value, reward, weight, gamma, lambda_)
    return td_lambda_fwd(value, reward, weight, float(gamma), float(lambda_))[0]


def upgo(logit, action, mask, rho, reward, value, TB, K, N):
    if not torch.compiler.is_compiling():
        ret = ops.lambda_returns_(value, reward, None, 1.0, None, 1.0, None, True)
        return ops.UPGOFunction.apply(logit, action, mask, rho, ret, value, TB, K, N)
    ret = lambda_returns(value, reward, None, 1.0, None, 1.0, None, True)
    return upgo_fwd(logit, action, mask, rho, ret, value, TB, K, N, _want_grad(logit))[0]


def vtrace(target_output, value, behaviour_output, action, reward, weight, gamma, lambda_, rho_clip, c_clip, rho_pg_clip):
    """-> (policy_loss, value_loss, entropy_loss), as VTraceFunction"""
    if not torch.compiler.is_compiling():
        return ops.VTraceFunction.apply(target_output, value, behaviour_output, action, reward, weight, gamma, lambda_,
                                        rho_clip, c_clip, rho_pg_clip)
    out = vtrace_loss(target_output, value, behaviour_output, action, reward, weight, gamma, lambda_, rho_clip, c_clip,
                      rho_pg_clip, _want_grad(target_output, value))[0]
    return out[0], out[1], out[2]


def ppo_value(value_new, value_old, return_, weight, clip_ratio, use_value_clip):
    if not torch.compiler.is_compiling():
        return ops.ppo_value_(value_new, value_old, return_, weight, clip_ratio, use_value_clip)
    return ppo_value_fwd(value_new, value_old, return_, weight, float(clip_ratio), bool(use_value_clip),
                         _want_grad(value_new))[0]


def token_logp(logits, index, dt):
    """-> log p(index) per row of logits (rows, V) staged by ``stage_logits``, as TokenLogProbFunction"""
    if not torch.compiler.is_compiling():
        return ops.TokenLogProbFunction.apply(logits, index, dt)
    return token_logp_op(logits, index)[0]


def lm_policy(logit_new, logit_old, logit_ref, action, side, weight, mode, dt, clip_ratio, beta):
    """-> (loss, approx_kl, clipfrac), as GRPOFunction (``mode`` 'grpo': side = adv (B)) or RLOOFunction ('rloo': side =
    reward (K, B / K), no logit_ref); logits staged by ``stage_logits``"""
    if not torch.compiler.is_compiling():
        if mode == 'grpo':
            return ops.GRPOFunction.apply(logit_new, logit_old, logit_ref, action, side, weight, dt, clip_ratio, beta)
        return ops.RLOOFunction.apply(logit_new, logit_old, action, side, weight, dt, clip_ratio)
    out = lm_policy_fwd(logit_new, logit_old, logit_ref, action, side, weight, mode, float(clip_ratio), float(beta))[0]
    return out[0], out[1], out[2]


def token_head(lp_new, lp_old, lp_ref, adv, reward, weight, clip_ratio, beta):
    """-> (loss, approx_kl, clipfrac), as ops.token_head_"""
    if not torch.compiler.is_compiling():
        return ops.token_head_(lp_new, lp_old, lp_ref, adv, reward, weight, clip_ratio, beta)
    out = token_head_fwd(lp_new, lp_old, lp_ref, adv, reward, weight, float(clip_ratio), float(beta))[0]
    return out[0], out[1], out[2]


def ppo_lm(logit_new, logit_old, logit_pre, action, adv, weight, dt, clip_ratio, dual_clip, kl_type, entropy, hint_kind):
    """-> (policy_loss, entropy_loss, kl_div, the five floats), as PPOLMFunction; logits staged by ``stage_logits``"""
    if not torch.compiler.is_compiling():
        return ops.PPOLMFunction.apply(logit_new, logit_old, logit_pre, action, adv, weight, dt, clip_ratio, dual_clip,
                                       kl_type, entropy, hint_kind)
    out = ppo_lm_fwd(logit_new, logit_old, logit_pre, action, adv, weight, clip_ratio, dual_clip, kl_type, entropy)[0]
    return out[0], out[1], out[2], out


def a2c_lm(logit, value, action, adv, return_, weight, dt):
    """-> (policy_loss, value_loss, entropy_loss), as A2CLMFunction; logit staged by ``stage_logits``"""
    if not torch.compiler.is_compiling():
        return ops.A2CLMFunction.apply(logit, value, action, adv, return_, weight, dt)
    out = a2c_lm_fwd(logit, value, action, adv, return_, weight)[0]
    return out[0], out[1], out[2]


def lm_logp(hidden, lm_weight, index, dt):
    """-> log p(index) per token row, as TokenLogpLinearFunction"""
    if torch.compiler.is_compiling():
        return lm_logp_op(hidden, lm_weight, index, dt)[0]
    if _want_grad(hidden, lm_weight):
        return ops.TokenLogpLinearFunction.apply(hidden, lm_weight, index, dt)
    return ops.lm_logp_fwd_(hidden.detach(), lm_weight.detach(), index, dt)[0]


def lm_linear_loss(hidden, lm_weight, action, lp_old, lp_ref, side, weight, kind, B, S, dt, clip_ratio, beta):
    """-> (loss, approx_kl, clipfrac), as LMLinearLossFunction"""
    if torch.compiler.is_compiling():
        grad = torch.is_grad_enabled()
        out = lm_linear_loss_op(hidden, lm_weight, action, lp_old, lp_ref, side, weight, kind, B, S, dt, clip_ratio, beta,
                                grad and hidden.requires_grad, grad and lm_weight.requires_grad)[0]
        return out[0], out[1].detach(), out[2].detach()
    if _want_grad(hidden, lm_weight):
        return ops.LMLinearLossFunction.apply(hidden, lm_weight, action, lp_old, lp_ref, side, weight, kind, B, S, dt,
                                              clip_ratio, beta)
    out = ops.lm_linear_loss_(hidden.detach(), lm_weight.detach(), action, lp_old, lp_ref, side, weight, kind, B, S, dt,
                              clip_ratio, beta, False, False)[0]
    return out[0], out[1], out[2]


def lm_linear_pg(hidden, lm_weight, value, action, adv, weight, lp_old, lp_pre, ret, kind, dt, cfg):
    """-> (the one loss, the raw sums), as LMLinearPGFunction"""
    grad = torch.is_grad_enabled()
    want = (grad and hidden.requires_grad, grad and lm_weight.requires_grad,
            grad and value is not None and value.requires_grad)
    if torch.compiler.is_compiling():
        return lm_linear_pg_op(hidden, lm_weight, value, action, adv, weight, lp_old, lp_pre, ret, kind, dt, *cfg,
                               *want)[:2]
    if any(want):
        return ops.LMLinearPGFunction.apply(hidden, lm_weight, value, action, adv, weight, lp_old, lp_pre, ret, kind, dt,
                                            cfg)
    out = ops.lm_linear_pg_(hidden.detach(), lm_weight.detach(), action, adv, weight, lp_old, lp_pre,
                            None if value is None else value.detach(), ret, kind, dt, cfg, False, False, False)[0]
    return ops.lm_pg_loss_(out, kind, cfg), out


def gae_returns(value, next_value, reward, done, traj_flag, gamma, lambda_, vscale):
    """-> (adv, unnormalized return, value_out or None, return_out or None, return_stats, adv_stats), as ops.gae_returns_"""
    if not torch.compiler.is_compiling():
        return ops.gae_returns_(value, next_value, reward, done, traj_flag, gamma, lambda_, 1, vscale, True, True,
                                want_adv_stats=True)
    adv, unnorm, vout, rout, stats, astats = gae_returns_op(value, next_value, reward, done, traj_flag, float(gamma),
                                                            float(lambda_), float(vscale))
    if vscale == 0.0:
        vout = rout = None
    return adv, unnorm, vout, rout, stats, astats


def ppof_gae_returns(value, next_value, reward, done, traj_flag, gamma, lambda_, value_norm, std, mu, sigma):
    """-> (adv, value_out, return_out, return_stats or None, adv_stats), as ops.gae_returns_norm_"""
    if not torch.compiler.is_compiling():
        return ops.gae_returns_norm_(value, next_value, reward, done, traj_flag, gamma, lambda_, value_norm, std, mu, sigma,
                                     value_norm == 'baseline')
    adv, vout, rout, stats, astats = gae_returns_norm(value, next_value, reward, done, traj_flag, float(gamma),
                                                      float(lambda_), value_norm, float(std), mu, sigma)
    return adv, vout, rout, stats if value_norm == 'baseline' else None, astats


def adv_stats(x):
    """{mean, std (unbiased) + 1e-8} of ``x``"""
    return adv_stats_op(x) if torch.compiler.is_compiling() else ops.adv_stats_(x)


def normalize(x, stats):
    return normalize_op(x, stats) if torch.compiler.is_compiling() else ops.normalize_(x, stats)


def value_map(x, mode):
    """symlog (``mode`` 0) or inv_symlog (1) of a contiguous fp32 tensor, differentiable"""
    return value_map_op(x, mode) if torch.compiler.is_compiling() else ops.ValueMapFunction.apply(x, mode)


def quantile_td(q, next_n_q, action, next_n_action, reward, done, tau, weight, value_gamma, vg_stride, B, N, n_tau,
                n_tau_prime, nstep, gamma, form, kappa):
    """-> (loss, td), as QuantileTDFunction; the layout of q / next_n_q is QUANTILE_AXES[form]"""
    if not torch.compiler.is_compiling():
        return ops.QuantileTDFunction.apply(q, next_n_q, action, next_n_action, reward, done, tau, weight,
                                            _const(value_gamma, q.device), vg_stride, B, N, n_tau, n_tau_prime, nstep,
                                            gamma, _quantile_strides(q, form), _quantile_strides(next_n_q, form),
                                            (tau.stride(0), tau.stride(1)), form, kappa)
    vg, vg_scalar = _scalar_or_tensor(value_gamma)
    loss, td, _, _ = quantile_fwd(q, next_n_q, action, next_n_action, reward, done, tau, weight, vg, vg_scalar, vg_stride,
                                  B, N, n_tau, n_tau_prime, nstep, gamma, form, kappa, _want_grad(q))
    return loss, td


def ppo_continuous(mu, sigma, value_new, mu_old, sigma_old, mu_pre, sigma_pre, action, value_old, adv, return_, weight, S,
                   D, clip_ratio, use_value_clip, dual_clip, kl_type, hint_kind, factor=None):
    """-> (policy, value, entropy, kl loss, a vector whose [4:6] are approx_kl, clipfrac), as PPOContinuousFunction"""
    if not torch.compiler.is_compiling():
        return ops.PPOContinuousFunction.apply(mu, sigma, value_new, mu_old, sigma_old, mu_pre, sigma_pre, action,
                                               value_old, adv, return_, weight, S, D, clip_ratio, use_value_clip,
                                               dual_clip, kl_type, hint_kind, factor)
    out = ppoc_loss(mu, sigma, value_new, mu_old, sigma_old, mu_pre, sigma_pre, action, value_old, adv, return_, weight,
                    factor, S, D, clip_ratio, use_value_clip, dual_clip, kl_type, hint_kind,
                    _want_grad(mu, sigma, value_new))[0]
    return out[0], out[1], out[2], out[3], out


def coma(logit, q_value, target_q, action, reward, weight, T, B, A, N, gamma, lambda_):
    """-> (policy_loss, q_value_loss, entropy_loss), as COMAFunction without the differentiable returns"""
    if not torch.compiler.is_compiling():
        return ops.COMAFunction.apply(logit, q_value, target_q, action, reward, weight, None, T, B, A, N, gamma, lambda_)
    out = coma_fwd(logit, q_value, target_q, action, reward, weight, T, B, A, N, float(gamma), float(lambda_),
                   _want_grad(logit, q_value))[0]
    return out[0], out[1], out[2]


def dqfd(q, next_n_q, next_q1, action, next_n_action, next_action1, reward, done, done1, weight, value_gamma, vg_stride,
         is_expert, S, N, nstep, gamma, cum_reward, rescale, eps, criterion, crit_param, lam_n, lam_1, lam_s, margin,
         seq_len, priority_mix, want_targets, want_priority):
    """-> (loss, td, s_n, s_1, s_je, tn, t1, prio), as DQfDTDFunction; value_gamma and is_expert may be python floats
    (is_expert then holds for all S rows)"""
    if not torch.compiler.is_compiling():
        dev = q.device
        ie = ops.const_scalar(is_expert, dev).expand(S).contiguous() if _is_scalar(is_expert) else is_expert
        return ops.DQfDTDFunction.apply(q, next_n_q, next_q1, action, next_n_action, next_action1, reward, done, done1,
                                        weight, _const(value_gamma, dev), vg_stride, ie, S, N, nstep, gamma, cum_reward,
                                        rescale, eps, criterion, crit_param, lam_n, lam_1, lam_s, margin, seq_len,
                                        priority_mix, want_targets, want_priority)
    vg, vg_scalar = _scalar_or_tensor(value_gamma)
    ie, ie_scalar = _scalar_or_tensor(is_expert)
    loss, td, stats, _, tn, t1, prio, _ = dqfd_fwd(
        q, next_n_q, next_q1, action, next_n_action, next_action1, reward, done, done1, weight, vg, vg_scalar, vg_stride,
        ie, ie_scalar, S, N, nstep, gamma, cum_reward, rescale, eps, criterion, crit_param, lam_n, lam_1, lam_s, margin,
        seq_len, priority_mix, want_targets, want_priority, _want_grad(q))
    s_n, s_1, s_je = stats.unbind(0)
    return loss, td, s_n, s_1, s_je, tn, t1, prio


def soft_td(q, target_q, next_q, action, reward, done, weight, value_gamma, vg_stride, mode, S, G, N, nstep, gamma, tau,
            alpha, cum_reward, criterion, crit_param):
    """-> (loss, td, target, action_gap, clipfrac, record_target_v), as SoftTDFunction"""
    if not torch.compiler.is_compiling():
        return ops.SoftTDFunction.apply(q, target_q, next_q, action, reward, done, weight, _const(value_gamma, q.device),
                                        vg_stride, mode, S, G, N, nstep, gamma, tau, alpha, cum_reward, criterion,
                                        crit_param)
    vg, vg_scalar = _scalar_or_tensor(value_gamma)
    loss, td, _, target, gap, clip, rec, _ = soft_td_fwd(q, target_q, next_q, action, reward, done, weight, vg, vg_scalar,
                                                         vg_stride, mode, S, G, N, nstep, gamma, tau, alpha, cum_reward,
                                                         criterion, crit_param, _want_grad(q))
    return loss, td, target, gap, clip, rec


def fqf_fraction(q_tau_i, q_value, quantiles, action, B, N):
    """-> the fraction loss, as FQFFractionFunction"""
    if not torch.compiler.is_compiling():
        return ops.FQFFractionFunction.apply(q_tau_i, q_value, quantiles, action, B, N, q_tau_i.stride(), q_value.stride(),
                                             quantiles.stride())
    return fqf_fraction_fwd(q_tau_i, q_value, quantiles, action, B, N, _want_grad(quantiles))[0]


def scatter(x, row, col, H, W, mode):
    """ScatterConnection's scatter of x (B, M, N) into (B, N, H, W), as ScatterFunction"""
    if not torch.compiler.is_compiling():
        return ops.ScatterFunction.apply(x, row, col, H, W, mode)
    return scatter_fwd(x, row, col, H, W, mode)


def lnlstm(x, h0, c0, wx, wh, bias, gamma_x, beta_x, gamma_h, beta_h, save):
    """one layer of the layer-normalised LSTM -> (y, h_T, c_T), as LNLSTMFunction; ``save`` when a gradient is wanted"""
    args = (x, h0, c0, wx, wh, bias, gamma_x, beta_x, gamma_h, beta_h)
    if torch.compiler.is_compiling():
        return lnlstm_fwd(*args, save)[:3]
    if not save:  # nothing to differentiate: no autograd node
        return ops.lnlstm_fwd_(*args, False)[:3]
    return ops.LNLSTMFunction.apply(*args, save)
