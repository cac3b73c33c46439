"""The hot-path launches of ``ops`` as ``torch.library`` custom ops (namespace ``b200rl``), so that ``torch.compile`` can
trace the eight operators of the reference's plugin boundary (gae, ppo_error, q_nstep_td_error,
q_nstep_td_error_with_rescale, dist_nstep_td_error, td_lambda_error, upgo_loss, vtrace_error_discrete_action) without a
graph break, and ``mode="reduce-overhead"`` can replay a compiled learner step as a CUDA graph.

Each op's implementation is the launch function ``ops`` runs in eager mode; ``rl_utils`` calls the wrappers at the bottom
of this module only while ``torch.compiler.is_compiling()``.  The schemas hold tensors and scalars only: the workspace, the
upstream-gradient records and cached constants are looked up inside the implementations, when the op runs.

The forward-written gradients work as in eager mode, with one difference that functional ops impose: a backward op may
not return its input, so after a forward launch that wrote the gradients the backward op copies them once and runs the
verify launch on the copy (recomputing on the device when the upstream gradients differ from the record, no host sync).
"""
from typing import Optional

import torch
from torch import Tensor

from . import ops


def _empty(like):
    return like.new_empty(0)


def _forward_grads(written, g_used, *grads):
    """copies of the forward-written gradients and their record, or None when the forward wrote none"""
    return tuple(g.clone() for g in grads) + (g_used, ) if written else None


def _upstream(g, n):
    """the device pointers of the first ``n`` floats of an upstream-gradient vector (None: no gradient, 0)"""
    if g is None:
        return None, (None, ) * n
    g = g.float().contiguous()
    base = g.data_ptr()
    return g, tuple(base + 4 * i for i in range(n))


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
    ctx.save_for_backward(*inputs[:11], *output[1:])
    ctx.cfg = inputs[11:19]
    ctx.mark_non_differentiable(*output[1:])


def _ppo_backward(ctx, g_out, *_):
    saved = ctx.saved_tensors
    if g_out is None:
        return (None, ) * 20
    grad_logit, grad_value = ppo_bwd(*saved[:11], g_out, *saved[11:], *ctx.cfg)
    return (grad_logit, grad_value) + (None, ) * 18


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
    skip = 1 if (g_td is None and grad_unit.numel()) else 0
    grad = grad_unit.clone() if skip else dcrit.new_empty(S * G, N)
    return ops.qntd_bwd_(dcrit, weight, action, pg, ptd, S, G, N, group_mean, 0, skip, grad)


@qntd_bwd.register_fake
def _(dcrit, weight, action, g_loss, g_td, grad_unit, S, G, N, group_mean):
    return dcrit.new_empty(S * G, N)


def _qntd_setup(ctx, inputs, output):
    q, action, weight = inputs[0], inputs[2], inputs[6]
    ctx.save_for_backward(output[2], weight, action, output[4])
    ctx.cfg = (inputs[11], inputs[12], inputs[13], inputs[21])
    ctx.q_shape = q.shape
    ctx.set_materialize_grads(False)
    ctx.mark_non_differentiable(*output[2:])


def _qntd_backward(ctx, g_loss, g_td, *_):
    if g_loss is None and g_td is None:
        return (None, ) * 23
    dcrit, weight, action, grad_unit = ctx.saved_tensors
    grad = qntd_bwd(dcrit, weight, action, g_loss, g_td, grad_unit, *ctx.cfg)
    return (grad.view(ctx.q_shape), ) + (None, ) * 22


qntd_fwd.register_autograd(_qntd_backward, setup_context=_qntd_setup)


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
    skip = 1 if (g_td is None and grad_unit.numel()) else 0
    grad = grad_unit.clone() if skip else torch.empty_like(dist)
    return ops.dntd_bwd_(dist, act, proj, weight, w_stride, pg, ptd, R, N, n_atom, skip, grad)


@dntd_bwd.register_fake
def _(dist, *args):
    return torch.empty_like(dist)


def _dntd_setup(ctx, inputs, output):
    ctx.save_for_backward(inputs[0], inputs[2], output[2], inputs[6], output[3])
    B, A, N, n_atom = inputs[12:16]
    ctx.cfg = (inputs[7], inputs[8], B * A, N, n_atom)
    ctx.set_materialize_grads(False)
    ctx.mark_non_differentiable(*output[2:])


def _dntd_backward(ctx, g_loss, g_td, *_):
    if g_loss is None and g_td is None:
        return (None, ) * 22
    dist, act, proj, weight, grad_unit = ctx.saved_tensors
    weight_scalar, w_stride, R, N, n_atom = ctx.cfg
    grad = dntd_bwd(dist, act, proj, weight, weight_scalar, w_stride, g_loss, g_td, grad_unit, R, N, n_atom)
    return (grad, ) + (None, ) * 21


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
    return scale(g_loss, dvalue), None, None, None, None


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
    skip = 1 if grad_unit.numel() else 0
    grad = grad_unit.clone() if skip else torch.empty_like(logit)
    kg, pg = _one(g_loss)
    return ops.upgo_bwd_(logit, action, mask, adv, pg, TB, K, N, skip, grad)


@upgo_bwd.register_fake
def _(logit, *args):
    return torch.empty_like(logit)


def _upgo_setup(ctx, inputs, output):
    ctx.save_for_backward(inputs[0], inputs[1], inputs[2], output[1], output[2])
    ctx.cfg = inputs[6:9]
    ctx.mark_non_differentiable(*output[1:])


def _upgo_backward(ctx, g_loss, *_):
    logit, action, mask, adv, grad_unit = ctx.saved_tensors
    return (upgo_bwd(logit, action, mask, adv, g_loss, grad_unit, *ctx.cfg), ) + (None, ) * 9


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
    ctx.save_for_backward(inputs[0], inputs[2], inputs[3], inputs[1], inputs[4], inputs[5], *output[1:])
    ctx.scal = inputs[6:11]
    ctx.mark_non_differentiable(*output[1:])


def _vtrace_backward(ctx, g_out, *_):
    if g_out is None:
        return (None, ) * 12
    grad_logit, grad_value = vtrace_bwd(*ctx.saved_tensors[:6], g_out, *ctx.saved_tensors[6:], *ctx.scal)
    return (grad_logit, grad_value) + (None, ) * 10


vtrace_loss.register_autograd(_vtrace_backward, setup_context=_vtrace_setup)


# ---------------------------------------------------------------------------------------------------------------------
# what rl_utils calls while compiling: the autograd.Function signatures of ops, on the ops above
# ---------------------------------------------------------------------------------------------------------------------
def _want_grad(*xs):
    return torch.is_grad_enabled() and any(x.requires_grad for x in xs)


def _scalar_or_tensor(x):
    """(tensor, None) or (None, python float): the custom ops take a python-scalar weight / value_gamma as a float"""
    return (None, float(x)) if (x is not None and not isinstance(x, Tensor)) else (x, None)


def ppo(logit_new, value_new, logit_old, action, value_old, adv, return_, weight, logit_pre, S, G, N, clip_ratio,
        use_value_clip, dual_clip, kl_type, hint_kind, adv_stats=None, factor=None):
    """-> the six floats policy, value, entropy, kl loss, approx_kl, clipfrac"""
    return ppo_loss(logit_new, value_new, logit_old, action, value_old, adv, return_, weight, logit_pre, adv_stats, factor,
                   S, G, N, clip_ratio, use_value_clip, dual_clip, kl_type, hint_kind,
                   _want_grad(logit_new, value_new))[0]


def qntd(q, next_n_q, action, next_n_action, reward, done, weight, value_gamma, vg_stride, gamma_ps, S, G, N, nstep, gamma,
         cum_reward, rescale, eps, criterion, crit_param, group_mean):
    """-> (loss, td, target), as QNStepTDFunction's first three outputs"""
    vg, vg_scalar = _scalar_or_tensor(value_gamma)
    loss, td, _, target, _ = qntd_fwd(q, next_n_q, action, next_n_action, reward, done, weight, vg, vg_scalar, vg_stride,
                                      gamma_ps, S, G, N, nstep, gamma, cum_reward, rescale, eps, criterion, crit_param,
                                      group_mean, _want_grad(q))
    return loss, td, target


def dist_nstep_td(dist, next_n_dist, act, next_n_act, reward, done, weight, w_stride, value_gamma, vg_stride, B, A, N,
                  n_atom, nstep, gamma, v_min, v_max, check_positive):
    """-> (loss, td)"""
    w, w_scalar = _scalar_or_tensor(weight)
    vg, vg_scalar = _scalar_or_tensor(value_gamma)
    loss, td, _, _ = dntd_fwd(dist, next_n_dist, act, next_n_act, reward, done, w, w_scalar, w_stride, vg, vg_scalar,
                              vg_stride, B, A, N, n_atom, nstep, gamma, v_min, v_max, check_positive, _want_grad(dist))
    return loss, td


def td_lambda(value, reward, weight, gamma, lambda_):
    return td_lambda_fwd(value, reward, weight, gamma, lambda_)[0]


def upgo(logit, action, mask, rho, reward, value, TB, K, N):
    ret = lambda_returns(value, reward, None, 1.0, None, 1.0, None, True)
    return upgo_fwd(logit, action, mask, rho, ret, value, TB, K, N, _want_grad(logit))[0]


def vtrace(target_output, value, behaviour_output, action, reward, weight, gamma, lambda_, rho_clip, c_clip, rho_pg_clip):
    """-> (policy_loss, value_loss, entropy_loss)"""
    out = vtrace_loss(target_output, value, behaviour_output, action, reward, weight, gamma, lambda_, rho_clip, c_clip,
                     rho_pg_clip, _want_grad(target_output, value))[0]
    return out[0], out[1], out[2]
