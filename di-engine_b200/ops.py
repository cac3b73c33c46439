"""Tensor-level operators over the C ABI (``include/b200rl.h``): allocation of outputs, stream / workspace plumbing and
``torch.autograd.Function`` wrappers.  torch is used for device memory, streams and autograd bookkeeping only; every
arithmetic step of the hot path runs in the CUDA kernels of ``csrc/``.

Nothing here computes on the CPU.  Host (CPU) tensors are accepted by the public API in ``rl_utils`` by staging them
to the current CUDA device and returning results on the host -- the "host buffers" end-to-end path.
"""
import os

import torch

from . import _lib

_WS = {}
_CONST = {}


def lib():
    return _lib.load()


def require_cuda():
    if not torch.cuda.is_available():
        raise _lib.B200RLError(
            "di_engine_b200 needs a CUDA device (sm_90a). There is no CPU implementation of the operators; "
            "the CPU oracle under oracle/ is test infrastructure only."
        )
    lib()


def stream_ptr():
    """raw cudaStream_t of torch's current stream on the current device (the fast private accessor when torch has it: the
    public ``torch.cuda.current_stream().cuda_stream`` costs noticeably more host time per call, and an operator asks twice)"""
    try:
        return torch._C._cuda_getCurrentRawStream(torch.cuda.current_device())
    except AttributeError:
        return torch.cuda.current_stream().cuda_stream


class _NoCtx:

    def __enter__(self):
        return None

    def __exit__(self, *a):
        return False


_NOCTX = _NoCtx()


def on_device(device):
    """``torch.cuda.device(device)`` only when ``device`` is not already current (entering the guard costs several
    microseconds of host time -- more than the launch it protects at the learner's real batch sizes)"""
    idx = device.index
    if idx is None or idx == torch.cuda.current_device():
        return _NOCTX
    return torch.cuda.device(device)


def workspace(device):
    """One zero-initialised scratch buffer per (device, stream): launches sharing it are stream-ordered."""
    idx = device.index
    if idx is None:
        idx = torch.cuda.current_device() if device.type == 'cuda' else -1
    key = (idx, stream_ptr())
    ws = _WS.get(key)
    if ws is None:
        nbytes = lib().b200rl_workspace_bytes()
        ws = torch.zeros(nbytes // 4, dtype=torch.float32, device=device)
        _WS[key] = ws
    return ws


def ptr(t):
    return None if t is None else t.data_ptr()


def f32c(t, name='tensor'):
    """fp32, contiguous; integer / bool flags (done, traj_flag, masks) are widened like the reference's ``.float()``."""
    if t is None:
        return None
    if t.dtype != torch.float32:
        if t.dtype in (torch.float64, torch.float16, torch.bfloat16):
            raise TypeError("di_engine_b200: %s must be float32 (got %s); the CUDA path computes in fp32" %
                            (name, t.dtype))
        t = t.float()
    return t if t.is_contiguous() else t.contiguous()


# B200RL_CHECK_INDICES=1 (or ops.CHECK_INDICES = True): every action / label tensor is range-checked on the host before its
# pointer goes to a kernel -- an out-of-range index raises IndexError as torch's gather would, at the price of one device
# synchronisation per call.  Off by default: the kernels index with the value they are given.
CHECK_INDICES = os.environ.get('B200RL_CHECK_INDICES', '0') == '1'


def i64c(t, n=None, name='action'):
    if t.dtype != torch.int64:
        t = t.long()
    if CHECK_INDICES and n is not None and t.numel():
        lo, hi = torch.aminmax(t)
        lo, hi = int(lo), int(hi)
        if lo < 0 or hi >= n:
            raise IndexError("di_engine_b200: %s holds index %d, out of range for %d classes" % (name, lo if lo < 0 else hi, n))
    return t if t.is_contiguous() else t.contiguous()


def to_device(t, device):
    if isinstance(t, torch.Tensor) and t.device != device:
        return t.to(device, non_blocking=True)
    return t


def compute_device(*tensors):
    """Device the op runs on: the device of the first CUDA tensor, else the current CUDA device (host-buffer path)."""
    require_cuda()
    for t in tensors:
        if isinstance(t, torch.Tensor) and t.is_cuda:
            return t.device
    return torch.device('cuda', torch.cuda.current_device())


def const_scalar(value, device):
    """A cached 1-element device tensor holding a python scalar (weights / value_gamma given as floats)."""
    key = (float(value), device.index)
    t = _CONST.get(key)
    if t is None:
        t = torch.full((1, ), float(value), dtype=torch.float32, device=device)
        _CONST[key] = t
    return t


def _grads(*grads):
    """Upstream gradients as contiguous fp32 tensors, to be kept alive across the launch, and their device pointers
    (None -> the kernel treats that gradient as 0)."""
    keep = [None if g is None else g.float().contiguous() for g in grads]
    return keep, [ptr(g) for g in keep]


# The forward launch of the wrappers below also writes the gradients for the upstream gradients it expects: the loss
# weights of the training loop, remembered on the device per call-site kind (a policy-only caller must not disturb its
# full loss's record) and started from these defaults.  The backward launch verifies them on the device and recomputes on
# a mismatch -- exact for any upstream gradient, no host sync.
_HINT_INIT = {
    'ppo': [1.0, 0.5, -0.01, 0.0],
    'happo': [1.0, 0.5, -0.01, 0.0],
    'a2c': [1.0, 0.5, -0.01, 0.0],
    'a2cc': [1.0, 0.5, -0.01, 0.0],
    'ppoc': [1.0, 0.5, -0.01, 0.0],
    'happoc': [1.0, 0.5, -0.01, 0.0],
    'policy': [1.0, 0.0, -0.01, 0.0],
    'happo_policy': [1.0, 0.0, -0.01, 0.0],
    'ppoc_policy': [1.0, 0.0, -0.01, 0.0],
    'vtrace': [1.0, 0.5, -0.01],
}
_HINT = {}


def head_hint(device, kind, init):
    """device-resident expectation of the upstream gradients of a loss head (one record per head kind and device)"""
    key = (device.index, kind)
    h = _HINT.get(key)
    if h is None:
        h = torch.tensor(init, dtype=torch.float32, device=device)
        _HINT[key] = h
    return h


def ppo_hint(device, kind='ppo'):
    """The record of call-site ``kind`` (a key of ``_HINT_INIT``): (d total/d policy_loss, d/d value_loss, d/d entropy_loss
    [, d/d kl_div])."""
    return head_hint(device, kind, _HINT_INIT[kind])


def vtrace_hint(device):
    return ppo_hint(device, 'vtrace')


def _forward_grads(ctx):
    """The gradient buffers the forward launch wrote (``ctx.spec``), handed out once.  The first backward takes them, and
    dropping ctx's reference lets autograd adopt them as .grad without a copy; any later backward gets None and must
    recompute into fresh buffers, since by then .grad may own the first ones."""
    spec, ctx.spec = ctx.spec, None
    return spec


def _unit_grad(ctx, other_grads, fresh):
    """For the backward launches that take ``skip_if_unit`` (TD family, UPGO): (the forward-written gradient for a unit
    upstream gradient, 1) when it is still there and no gradient arrived through an output other than the loss; else
    (fresh(), 0), and the launch recomputes."""
    grad = _forward_grads(ctx)
    if grad is not None and all(g is None for g in other_grads):
        return grad, 1
    return fresh(), 0


# ----------------------------------------------------------------------------------------------------------------
# gae
# ----------------------------------------------------------------------------------------------------------------
def gae_(value, next_value, reward, done, traj_flag, gamma, lambda_, agents, mask_inplace=True):
    """value/next_value (T, C) contiguous fp32 CUDA; reward/done/traj (T, C/agents). next_value is masked in place."""
    T = value.shape[0]
    C = value.numel() // T if T > 0 else 0
    adv = torch.empty_like(value)
    if value.numel() == 0:
        return adv
    if C == 1 and agents == 1:
        # ONE sequence (the real PPO learner, ding/policy/ppo.py:280-282: n_sample steps of concatenated trajectories): the
        # segment-parallel single-CTA kernel of csrc/policy.cu instead of one lane walking all T steps
        return gae_returns_(value, next_value, reward, done, traj_flag, gamma, lambda_, 1, 0.0, False, False, mask_inplace)[0]
    with on_device(value.device):
        rc = lib().b200rl_gae(
            ptr(value), ptr(next_value), ptr(reward), ptr(done), ptr(traj_flag), ptr(adv), T, C, agents, float(gamma),
            float(lambda_), 1 if mask_inplace else 0, stream_ptr()
        )
    _lib.check(rc, 'b200rl_gae')
    return adv


def gae_returns_(value, next_value, reward, done, traj_flag, gamma, lambda_, agents, vscale, want_returns, want_stats,
                 mask_inplace=False, want_adv_stats=False):
    """gae + the pieces around it in PPOPolicy._forward_learn (ding/policy/ppo.py:274-297) -- csrc/policy.cu.
    -> (adv, unnormalized_return, value_out, return_out, stats3[, adv_stats2]) (None where not requested)."""
    T = value.shape[0]
    C = value.numel() // T
    dev = value.device
    adv = torch.empty_like(value)
    unnorm = torch.empty_like(value) if want_returns else None
    vout = torch.empty_like(value) if (want_returns and vscale != 0.0) else None
    rout = torch.empty_like(value) if (want_returns and vscale != 0.0) else None
    stats = torch.empty(3, dtype=torch.float32, device=dev) if want_stats else None
    astats = torch.empty(2, dtype=torch.float32, device=dev) if want_adv_stats else None
    with on_device(dev):
        ws = workspace(dev)
        rc = lib().b200rl_gae_returns(
            ptr(value), ptr(next_value), ptr(reward), ptr(done), ptr(traj_flag), T, C, agents, float(gamma), float(lambda_),
            1 if mask_inplace else 0, float(vscale), ptr(adv), ptr(unnorm), ptr(vout), ptr(rout), ptr(stats), ptr(astats),
            ptr(ws), ws.numel() * 4, stream_ptr()
        )
    _lib.check(rc, 'b200rl_gae_returns')
    if want_adv_stats:
        return adv, unnorm, vout, rout, stats, astats
    return adv, unnorm, vout, rout, stats


def adv_stats_(x):
    """{mean, std(unbiased) + 1e-8} of ``x`` as two device floats (ding/policy/ppo.py:304-306), one launch."""
    out = torch.empty(2, dtype=torch.float32, device=x.device)
    with on_device(x.device):
        ws = workspace(x.device)
        rc = lib().b200rl_adv_stats(ptr(x), x.numel(), ptr(out), ptr(ws), ws.numel() * 4, stream_ptr())
    _lib.check(rc, 'b200rl_adv_stats')
    return out


def normalize_(x, stats):
    out = torch.empty_like(x)
    with on_device(x.device):
        rc = lib().b200rl_normalize(ptr(x), ptr(stats), x.numel(), ptr(out), stream_ptr())
    _lib.check(rc, 'b200rl_normalize')
    return out


# ----------------------------------------------------------------------------------------------------------------
# ppo
# ----------------------------------------------------------------------------------------------------------------
# True: the forward pass also writes the gradients for the expected upstream gradients (``ppo_hint``), verified by the
# backward pass.  False: separate backward kernel always.
PPO_FUSED_BACKWARD = True


class PPOFunction(torch.autograd.Function):
    """Outputs: policy_loss, value_loss, entropy_loss, kl_div (differentiable 0-dim) and the raw 8-float result vector
    (non differentiable; [4]=approx_kl, [5]=clipfrac)."""

    @staticmethod
    def forward(ctx, logit_new, value_new, logit_old, action, value_old, adv, return_, weight, logit_pre, S, G, N,
                clip_ratio, use_value_clip, dual_clip, kl_type, hint_kind, adv_stats=None, factor=None):
        dev = logit_new.device
        ctx.hint_kind = hint_kind
        ctx.adv_stats = adv_stats  # {mean, std + 1e-8} device floats or None; kept alive for the backward launch
        ctx.factor = factor        # happo_error's per-sample factor (S,) or None; likewise
        out = torch.empty(8, dtype=torch.float32, device=dev)
        L = lib()
        tensors = (ptr(logit_new), ptr(logit_old), ptr(logit_pre), ptr(action), ptr(value_new), ptr(value_old),
                   ptr(adv), ptr(return_), ptr(weight))
        cfg = (S, G, N, clip_ratio, use_value_clip, dual_clip, kl_type, ptr(adv_stats), ptr(factor))
        ctx.spec = None
        want_grad = PPO_FUSED_BACKWARD and (ctx.needs_input_grad[0] or ctx.needs_input_grad[1])
        with on_device(dev):
            ws = workspace(dev)
            if want_grad:
                grad_logit = torch.empty_like(logit_new)
                grad_value = torch.empty_like(value_new)
                if L.b200rl_ppo_fused_supported(*tensors, ptr(grad_logit), G, N):
                    g_used = torch.empty(4, dtype=torch.float32, device=dev)
                    rc = L.b200rl_ppo_fwd_grad(*tensors, *cfg, ptr(ppo_hint(dev, hint_kind)), ptr(g_used), ptr(out),
                                               ptr(grad_logit), ptr(grad_value), ptr(ws), ws.numel() * 4,
                                               stream_ptr())
                    _lib.check(rc, 'b200rl_ppo_fwd_grad')
                    ctx.spec = (grad_logit, grad_value, g_used)
            if ctx.spec is None:
                rc = L.b200rl_ppo_fwd(*tensors, *cfg, ptr(out), ptr(ws), ws.numel() * 4, stream_ptr())
                _lib.check(rc, 'b200rl_ppo_fwd')
        ctx.save_for_backward(logit_new, value_new, logit_old, action, value_old, adv, return_, weight, logit_pre)
        ctx.cfg = cfg
        ctx.mark_non_differentiable(out)
        p, v, e, k = out[0], out[1], out[2], out[3]
        return p, v, e, k, out

    @staticmethod
    def backward(ctx, g_p, g_v, g_e, g_k, _g_out):
        logit_new, value_new, logit_old, action, value_old, adv, return_, weight, logit_pre = ctx.saved_tensors
        dev = logit_new.device
        keep, (pp, pv, pe, pk) = _grads(g_p, g_v, g_e, g_k)
        spec = _forward_grads(ctx)
        if spec is not None:  # valid if the expectation held; the kernel checks on the device
            grad_logit, grad_value, g_used = spec
            p_used, p_hint = ptr(g_used), ptr(ppo_hint(dev, ctx.hint_kind))
        else:  # no fused forward, or a repeated backward: null g_used / hint -> the kernel recomputes
            grad_logit = torch.empty_like(logit_new)
            grad_value = torch.empty_like(value_new)
            p_used, p_hint = None, None
        with on_device(dev):
            rc = lib().b200rl_ppo_bwd(
                ptr(logit_new), ptr(logit_old), ptr(logit_pre), ptr(action), ptr(value_new), ptr(value_old), ptr(adv),
                ptr(return_), ptr(weight), *ctx.cfg, pp, pv, pe, pk, p_used, p_hint, ptr(grad_logit), ptr(grad_value),
                stream_ptr()
            )
        _lib.check(rc, 'b200rl_ppo_bwd')
        return (grad_logit, grad_value) + (None, ) * 17


class GAEPPOFunction(torch.autograd.Function):
    """gae -> ppo_error in one launch (csrc/fused.cu).  Outputs: adv (T,B; non differentiable), the four losses and the
    raw result vector; backward is the same device-verified scheme as PPOFunction."""

    @staticmethod
    def forward(ctx, logit_new, value_new, value, next_value, reward, done, traj_flag, logit_old, action, value_old,
                return_, weight, logit_pre, T, B, N, gamma, lambda_, clip_ratio, use_value_clip, dual_clip, kl_type):
        dev = logit_new.device
        ctx.hint_kind = 'ppo'
        out = torch.empty(8, dtype=torch.float32, device=dev)
        adv = torch.empty_like(value)
        want_grad = ctx.needs_input_grad[0] or ctx.needs_input_grad[1]
        grad_logit = torch.empty_like(logit_new) if want_grad else None
        grad_value = torch.empty_like(value_new) if want_grad else None
        g_used = torch.empty(4, dtype=torch.float32, device=dev) if want_grad else None
        with on_device(dev):
            ws = workspace(dev)
            rc = lib().b200rl_gae_ppo_fwd_grad(
                ptr(value), ptr(next_value), ptr(reward), ptr(done), ptr(traj_flag), T, B, gamma, lambda_, 1,
                ptr(logit_new), ptr(logit_old), ptr(logit_pre), ptr(action), ptr(value_new), ptr(value_old),
                ptr(return_), ptr(weight), N, clip_ratio, use_value_clip, dual_clip, kl_type,
                ptr(ppo_hint(dev, ctx.hint_kind)) if want_grad else None, ptr(g_used), ptr(adv), ptr(out),
                ptr(grad_logit), ptr(grad_value), ptr(ws), ws.numel() * 4, stream_ptr()
            )
        _lib.check(rc, 'b200rl_gae_ppo_fwd_grad')
        ctx.save_for_backward(logit_new, value_new, logit_old, action, value_old, adv, return_, weight, logit_pre)
        ctx.cfg = (T * B, 1, N, clip_ratio, use_value_clip, dual_clip, kl_type, None, None)  # no adv_stats, no factor
        ctx.spec = (grad_logit, grad_value, g_used) if want_grad else None
        ctx.mark_non_differentiable(out, adv)
        return adv, out[0], out[1], out[2], out[3], out

    @staticmethod
    def backward(ctx, _g_adv, g_p, g_v, g_e, g_k, _g_out):
        grads = PPOFunction.backward(ctx, g_p, g_v, g_e, g_k, None)
        return (grads[0], grads[1]) + (None, ) * 20


def ppo_value_(value_new, value_old, return_, weight, clip_ratio, use_value_clip):
    """ppo_value_error (ppo.py:233-275): loss and, if needed, its gradient for a unit upstream gradient in one launch."""
    dev = value_new.device
    loss = torch.empty((), dtype=torch.float32, device=dev)
    want_grad = value_new.requires_grad and torch.is_grad_enabled()
    dvalue = torch.empty_like(value_new) if want_grad else None
    with on_device(dev):
        ws = workspace(dev)
        rc = lib().b200rl_ppo_value_fwd(
            ptr(value_new), ptr(value_old), ptr(return_), ptr(weight), value_new.numel(), float(clip_ratio),
            1 if use_value_clip else 0, ptr(loss), ptr(dvalue), ptr(ws), ws.numel() * 4, stream_ptr()
        )
    _lib.check(rc, 'b200rl_ppo_value_fwd')
    if want_grad:
        return _ScaleSaved.apply(value_new, loss, dvalue)
    return loss


def ppg_bc_(logit_new, logit_old, action):
    """behavioural-cloning term of ppg_joint_error (ppg.py:62-67): value (NaN-propagating, as the reference) and gradient."""
    dev = logit_new.device
    B, N = logit_new.shape
    loss = torch.empty((), dtype=torch.float32, device=dev)
    want_grad = logit_new.requires_grad and torch.is_grad_enabled()
    dlogit = torch.empty_like(logit_new) if want_grad else None
    with on_device(dev):
        ws = workspace(dev)
        rc = lib().b200rl_ppg_bc_fwd(ptr(logit_new), ptr(logit_old), ptr(action), B, N, ptr(loss), ptr(dlogit), ptr(ws),
                                     ws.numel() * 4, stream_ptr())
    _lib.check(rc, 'b200rl_ppg_bc_fwd')
    if want_grad:
        return _ScaleSaved.apply(logit_new, loss, dlogit)
    return loss


# ----------------------------------------------------------------------------------------------------------------
# q n-step TD
# ----------------------------------------------------------------------------------------------------------------
class QNStepTDFunction(torch.autograd.Function):
    """Outputs: loss and td_error_per_sample (both differentiable w.r.t. q, like the reference's, td.py:718-719), the
    detached n-step target and (sequence form) the priority mix (non differentiable).

    ONE forward launch also writes d loss / d q for a unit upstream gradient; ``backward`` hands that buffer to autograd
    after a verification launch that returns at once when the upstream gradient really was 1 (and no gradient arrived
    through td_error_per_sample), and recomputes otherwise -- exact for any upstream gradient, no host sync."""

    @staticmethod
    def forward(ctx, q, next_n_q, action, next_n_action, reward, done, weight, value_gamma, vg_stride, gamma_ps, S, G,
                N, nstep, gamma, cum_reward, rescale, eps, criterion, crit_param, group_mean, seq_len, priority_mix,
                want_priority):
        dev = q.device
        R = S * G
        loss = torch.empty((), dtype=torch.float32, device=dev)
        td = torch.empty(S if group_mean else R, dtype=torch.float32, device=dev)
        dcrit = torch.empty(R, dtype=torch.float32, device=dev)
        target = torch.empty(R, dtype=torch.float32, device=dev)
        prio = torch.empty(S // seq_len, dtype=torch.float32, device=dev) if want_priority else None
        grad_unit = torch.empty(R, N, dtype=torch.float32, device=dev) if ctx.needs_input_grad[0] else None
        with on_device(dev):
            ws = workspace(dev)
            rc = lib().b200rl_qntd_fwd(
                ptr(q), ptr(next_n_q), ptr(action), ptr(next_n_action), ptr(reward), ptr(done), ptr(weight),
                ptr(value_gamma), vg_stride, ptr(gamma_ps), S, G, N, nstep, gamma, cum_reward, rescale, eps, criterion,
                crit_param, group_mean, seq_len, priority_mix, ptr(loss), ptr(td), ptr(dcrit), ptr(target),
                ptr(grad_unit), ptr(prio), ptr(ws), ws.numel() * 4, stream_ptr()
            )
        _lib.check(rc, 'b200rl_qntd_fwd')
        ctx.save_for_backward(dcrit, action, weight)
        ctx.cfg = (S, G, N, group_mean, seq_len)
        ctx.q_shape = q.shape
        ctx.spec = grad_unit
        ctx.set_materialize_grads(False)
        if prio is None:
            prio = torch.empty(0, dtype=torch.float32, device=dev)
        ctx.mark_non_differentiable(target, prio)
        return loss, td, target, prio

    @staticmethod
    def backward(ctx, g_loss, g_td, _g_target, _g_prio):
        if g_loss is None and g_td is None:
            return (None, ) * 24
        dcrit, action, weight = ctx.saved_tensors
        S, G, N, group_mean, seq_len = ctx.cfg
        keep, (pg, ptd) = _grads(g_loss, g_td)
        grad_q, skip = _unit_grad(ctx, (g_td, ), lambda: torch.empty(S * G, N, dtype=torch.float32, device=dcrit.device))
        with on_device(dcrit.device):
            rc = lib().b200rl_qntd_bwd(ptr(dcrit), ptr(weight), ptr(action), pg, ptd, S, G, N, group_mean, seq_len, skip,
                                       ptr(grad_q), stream_ptr())
        _lib.check(rc, 'b200rl_qntd_bwd')
        return (grad_q.view(ctx.q_shape), ) + (None, ) * 23


class DQfDTDFunction(torch.autograd.Function):
    """DQfD n-step + 1-step TD + supervised margin loss (csrc/td.cu dqfd_fwd / dqfd_bwd).  Outputs: loss,
    td_error_per_sample and the three loss statistics (all differentiable w.r.t. q, as in the reference, td.py:974-983), the
    two detached targets and (sequence form) the priority mix (non differentiable).

    As QNStepTDFunction: ONE forward launch also writes d loss / d q for a unit upstream gradient, which ``backward`` hands
    to autograd after a verification launch; any other upstream gradient mix is recomputed on the device.  No host sync."""

    @staticmethod
    def forward(ctx, q, next_n_q, next_q1, action, next_n_action, next_action1, reward, done, done1, weight, value_gamma,
                vg_stride, is_expert, S, N, nstep, gamma, cum_reward, rescale, eps, criterion, crit_param, lam_n, lam_1,
                lam_s, margin, seq_len, priority_mix, want_targets, want_priority):
        dev = q.device
        loss = torch.empty((), dtype=torch.float32, device=dev)
        td = torch.empty(S, dtype=torch.float32, device=dev)
        stats = torch.empty(3, dtype=torch.float32, device=dev)
        saved = torch.empty(S, 4, dtype=torch.float32, device=dev)
        tn = torch.empty(S, dtype=torch.float32, device=dev) if want_targets else None
        t1 = torch.empty(S, dtype=torch.float32, device=dev) if want_targets else None
        prio = torch.empty(S // seq_len, dtype=torch.float32, device=dev) if want_priority else None
        grad_unit = torch.empty(S, N, dtype=torch.float32, device=dev) if ctx.needs_input_grad[0] else None
        with on_device(dev):
            ws = workspace(dev)
            rc = lib().b200rl_dqfd_fwd(
                ptr(q), ptr(next_n_q), ptr(next_q1), ptr(action), ptr(next_n_action), ptr(next_action1), ptr(reward),
                ptr(done), ptr(done1), ptr(weight), ptr(value_gamma), vg_stride, ptr(is_expert), S, N, nstep, gamma,
                cum_reward, rescale, eps, criterion, crit_param, lam_n, lam_1, lam_s, margin, seq_len, priority_mix,
                ptr(loss), ptr(td), ptr(stats), ptr(saved), ptr(tn), ptr(t1), ptr(grad_unit), ptr(prio), ptr(ws),
                ws.numel() * 4, stream_ptr()
            )
        _lib.check(rc, 'b200rl_dqfd_fwd')
        ctx.save_for_backward(saved, action, weight)
        ctx.cfg = (S, N, lam_n, lam_1, lam_s, seq_len)
        ctx.q_shape = q.shape
        ctx.spec = grad_unit
        ctx.set_materialize_grads(False)
        empty = torch.empty(0, dtype=torch.float32, device=dev)
        tn, t1, prio = (x if x is not None else empty for x in (tn, t1, prio))
        ctx.mark_non_differentiable(tn, t1, prio)
        s_n, s_1, s_je = stats.unbind(0)
        return loss, td, s_n, s_1, s_je, tn, t1, prio

    @staticmethod
    def backward(ctx, g_loss, g_td, g_sn, g_s1, g_sje, _g_tn, _g_t1, _g_prio):
        n_in = 30
        if g_loss is None and g_td is None and g_sn is None and g_s1 is None and g_sje is None:
            return (None, ) * n_in
        saved, action, weight = ctx.saved_tensors
        S, N, lam_n, lam_1, lam_s, seq_len = ctx.cfg
        keep, (pg, ptd, psn, ps1, psje) = _grads(g_loss, g_td, g_sn, g_s1, g_sje)
        grad_q, skip = _unit_grad(ctx, (g_td, g_sn, g_s1, g_sje),
                                  lambda: torch.empty(S, N, dtype=torch.float32, device=saved.device))
        with on_device(saved.device):
            rc = lib().b200rl_dqfd_bwd(ptr(saved), ptr(weight), ptr(action), pg, ptd, psn, ps1, psje, S, N, lam_n, lam_1,
                                       lam_s, seq_len, skip, ptr(grad_q), stream_ptr())
        _lib.check(rc, 'b200rl_dqfd_bwd')
        return (grad_q.view(ctx.q_shape), ) + (None, ) * (n_in - 1)


class SoftTDFunction(torch.autograd.Function):
    """The TD losses of the entropy-regularised value learners (csrc/td.cu soft_td_fwd): mode 0 Munchausen, 1 soft n-step
    (SQL), 2 value 1-step (discrete SAC).  Outputs: loss and td_error_per_sample (R rows; both differentiable w.r.t. q), the
    detached target, and the mode's statistics, which carry no gradient as in the reference: action_gap and clipfrac
    (mode 0), record_target_v (mode 1); the others are empty.

    Every target is detached, so the gradient reaches q through q_sa alone and the backward is QNStepTDFunction's launch
    (b200rl_qntd_bwd with G = 1 over the R rows).  As there, ONE forward launch also writes d loss / d q for a unit upstream
    gradient, which the backward verifies on the device and hands to autograd.  No host sync."""

    @staticmethod
    def forward(ctx, q, target_q, next_q, action, reward, done, weight, value_gamma, vg_stride, mode, S, G, N, nstep, gamma,
                tau, alpha, cum_reward, criterion, crit_param):
        dev = q.device
        R = S * G
        loss = torch.empty((), dtype=torch.float32, device=dev)
        td = torch.empty(R, dtype=torch.float32, device=dev)
        dcrit = torch.empty(R, dtype=torch.float32, device=dev)
        target = torch.empty(R, dtype=torch.float32, device=dev)
        gap = torch.empty((), dtype=torch.float32, device=dev) if mode == 0 else None
        clip = torch.empty(R, dtype=torch.float32, device=dev) if mode == 0 else None
        rec = torch.empty(R, dtype=torch.float32, device=dev) if mode == 1 else None
        grad_unit = torch.empty(R, N, dtype=torch.float32, device=dev) if ctx.needs_input_grad[0] else None
        with on_device(dev):
            ws = workspace(dev)
            rc = lib().b200rl_soft_td_fwd(
                mode, ptr(q), ptr(target_q), ptr(next_q), ptr(action), ptr(reward), ptr(done), ptr(weight),
                ptr(value_gamma), vg_stride, S, G, N, nstep, gamma, tau, alpha, cum_reward, criterion, crit_param,
                ptr(loss), ptr(td), ptr(dcrit), ptr(target), ptr(grad_unit), ptr(gap), ptr(clip), ptr(rec), ptr(ws),
                ws.numel() * 4, stream_ptr()
            )
        _lib.check(rc, 'b200rl_soft_td_fwd')
        ctx.save_for_backward(dcrit, action, weight)
        ctx.cfg = (R, 1, N, 0, 0)  # QNStepTDFunction's (S, G, N, group_mean, seq_len): R rows of one
        ctx.q_shape = q.shape
        ctx.spec = grad_unit
        ctx.set_materialize_grads(False)
        empty = torch.empty(0, dtype=torch.float32, device=dev)
        gap, clip, rec = (x if x is not None else empty for x in (gap, clip, rec))
        ctx.mark_non_differentiable(target, gap, clip, rec)
        return loss, td, target, gap, clip, rec

    @staticmethod
    def backward(ctx, g_loss, g_td, _g_target, _g_gap, _g_clip, _g_rec):
        return QNStepTDFunction.backward(ctx, g_loss, g_td, None, None)[:1] + (None, ) * 19


# ----------------------------------------------------------------------------------------------------------------
# ACER heads (csrc/acer.cu): un-reduced per-transition losses, plain forward / backward launches
# ----------------------------------------------------------------------------------------------------------------
class AcerPolicyFunction(torch.autograd.Function):
    """(actor_loss, bias_correction_loss), each (M,); differentiable w.r.t. target_logit only (acer.py:44-56)."""

    @staticmethod
    def forward(ctx, target_logit, q_values, q_retraces, v_pred, actions, ratio, M, N, c_clip_ratio):
        dev = target_logit.device
        actor = torch.empty(M, dtype=torch.float32, device=dev)
        bias = torch.empty(M, dtype=torch.float32, device=dev)
        with on_device(dev):
            rc = lib().b200rl_acer_policy_fwd(ptr(q_values), ptr(q_retraces), ptr(v_pred), ptr(target_logit), ptr(actions),
                                              ptr(ratio), M, N, c_clip_ratio, ptr(actor), ptr(bias), stream_ptr())
        _lib.check(rc, 'b200rl_acer_policy_fwd')
        ctx.save_for_backward(target_logit, q_values, q_retraces, v_pred, actions, ratio)
        ctx.cfg = (M, N, c_clip_ratio)
        ctx.set_materialize_grads(False)
        return actor, bias

    @staticmethod
    def backward(ctx, g_actor, g_bias):
        if g_actor is None and g_bias is None:
            return (None, ) * 9
        target_logit, q_values, q_retraces, v_pred, actions, ratio = ctx.saved_tensors
        M, N, c = ctx.cfg
        ga = f32c(g_actor) if g_actor is not None else None
        gb = f32c(g_bias) if g_bias is not None else None
        grad = torch.empty_like(target_logit)
        with on_device(target_logit.device):
            rc = lib().b200rl_acer_policy_bwd(ptr(q_values), ptr(q_retraces), ptr(v_pred), ptr(target_logit), ptr(actions),
                                              ptr(ratio), ptr(ga), ptr(gb), M, N, c, ptr(grad), stream_ptr())
        _lib.check(rc, 'b200rl_acer_policy_bwd')
        return (grad, ) + (None, ) * 8


class AcerValueFunction(torch.autograd.Function):
    """critic_loss (M,) = 0.5 (q_retraces - q_values[a])^2; differentiable w.r.t. q_values (acer.py:81-82)."""

    @staticmethod
    def forward(ctx, q_values, q_retraces, actions, M, N):
        loss = torch.empty(M, dtype=torch.float32, device=q_values.device)
        with on_device(q_values.device):
            rc = lib().b200rl_acer_value_fwd(ptr(q_values), ptr(q_retraces), ptr(actions), M, N, ptr(loss), stream_ptr())
        _lib.check(rc, 'b200rl_acer_value_fwd')
        ctx.save_for_backward(q_values, q_retraces, actions)
        ctx.cfg = (M, N)
        return loss

    @staticmethod
    def backward(ctx, g):
        q_values, q_retraces, actions = ctx.saved_tensors
        M, N = ctx.cfg
        gg = f32c(g)
        grad = torch.empty_like(q_values)
        with on_device(q_values.device):
            rc = lib().b200rl_acer_value_bwd(ptr(q_values), ptr(q_retraces), ptr(actions), ptr(gg), M, N, ptr(grad),
                                             stream_ptr())
        _lib.check(rc, 'b200rl_acer_value_bwd')
        return grad, None, None, None, None


def acer_trust_region_(grad, avg_logit, delta):
    N = grad.shape[-1]
    M = grad.numel() // N
    out = torch.empty_like(grad)
    with on_device(grad.device):
        rc = lib().b200rl_acer_trust_region(ptr(grad), ptr(avg_logit), M, N, float(delta), ptr(out), stream_ptr())
    _lib.check(rc, 'b200rl_acer_trust_region')
    return out


# ----------------------------------------------------------------------------------------------------------------
# quantile-regression n-step TD (QR-DQN / IQN / FQF)
# ----------------------------------------------------------------------------------------------------------------
class QuantileTDFunction(torch.autograd.Function):
    """loss and the per-sample losses (both differentiable w.r.t. q, as in the reference, td.py:1166,:1346,:1436); the forward
    launch also writes d loss / d q for a unit upstream gradient (verified on the device by the backward launch, as
    QNStepTDFunction).  ``q_strides`` / ``nq_strides`` / ``tau_strides``: element strides of (sample, quantile[, action])."""

    @staticmethod
    def forward(ctx, q, next_n_q, action, next_n_action, reward, done, tau, weight, value_gamma, vg_stride, B, N, n_tau,
                n_tau_prime, nstep, gamma, q_strides, nq_strides, tau_strides, form, kappa):
        dev = q.device
        loss = torch.empty((), dtype=torch.float32, device=dev)
        td = torch.empty(B, dtype=torch.float32, device=dev)
        dtheta = torch.empty(B, n_tau, dtype=torch.float32, device=dev)
        grad_unit = torch.empty_like(q) if ctx.needs_input_grad[0] else None
        with on_device(dev):
            ws = workspace(dev)
            rc = lib().b200rl_quantile_td_fwd(
                ptr(q), ptr(next_n_q), ptr(action), ptr(next_n_action), ptr(reward), ptr(done), ptr(tau), ptr(weight),
                ptr(value_gamma), vg_stride, B, N, n_tau, n_tau_prime, nstep, gamma, *q_strides, *nq_strides, *tau_strides,
                form, kappa, ptr(loss), ptr(td), ptr(dtheta), ptr(grad_unit), ptr(ws), ws.numel() * 4, stream_ptr()
            )
        _lib.check(rc, 'b200rl_quantile_td_fwd')
        ctx.save_for_backward(dtheta, action, weight)
        ctx.cfg = (B, N, n_tau, q_strides)
        ctx.q_shape = q.shape
        ctx.spec = grad_unit
        ctx.set_materialize_grads(False)
        return loss, td

    @staticmethod
    def backward(ctx, g_loss, g_td):
        if g_loss is None and g_td is None:
            return (None, ) * 21
        dtheta, action, weight = ctx.saved_tensors
        B, N, n_tau, q_strides = ctx.cfg
        keep, (pg, ptd) = _grads(g_loss, g_td)
        grad_q, skip = _unit_grad(ctx, (g_td, ),
                                  lambda: torch.empty(ctx.q_shape, dtype=torch.float32, device=dtheta.device))
        with on_device(dtheta.device):
            rc = lib().b200rl_quantile_td_bwd(ptr(dtheta), ptr(weight), ptr(action), pg, ptd, B, N, n_tau,
                                              *q_strides, skip, ptr(grad_q), stream_ptr())
        _lib.check(rc, 'b200rl_quantile_td_bwd')
        return (grad_q, ) + (None, ) * 20


class FQFFractionFunction(torch.autograd.Function):
    """FQF's fraction loss (td.py:1466-1513), differentiable w.r.t. ``quantiles`` only (q_tau_i and q_value enter detached,
    as the reference gathers them under no_grad); the forward launch also writes d loss / d quantiles for a unit upstream
    gradient (verified on the device by the backward launch, as QuantileTDFunction).  ``*_strides``: element strides of
    (sample, quantile[, action])."""

    @staticmethod
    def forward(ctx, q_tau_i, q_value, quantiles, action, B, N, qt_strides, qv_strides, qn_strides):
        dev = quantiles.device
        loss = torch.empty((), dtype=torch.float32, device=dev)
        g = torch.empty(B, N - 1, dtype=torch.float32, device=dev)
        grad_unit = torch.empty(B, N + 1, dtype=torch.float32, device=dev) if ctx.needs_input_grad[2] else None
        with on_device(dev):
            ws = workspace(dev)
            rc = lib().b200rl_fqf_fraction_fwd(
                ptr(q_tau_i), ptr(q_value), ptr(quantiles), ptr(action), B, N, q_tau_i.shape[2], q_value.shape[2],
                *qt_strides, *qv_strides, *qn_strides, ptr(loss), ptr(g), ptr(grad_unit), ptr(ws), ws.numel() * 4,
                stream_ptr()
            )
        _lib.check(rc, 'b200rl_fqf_fraction_fwd')
        ctx.save_for_backward(g)
        ctx.cfg = (B, N)
        ctx.spec = grad_unit
        ctx.set_materialize_grads(False)
        return loss

    @staticmethod
    def backward(ctx, g_loss):
        if g_loss is None:
            return (None, ) * 9
        g, = ctx.saved_tensors
        B, N = ctx.cfg
        keep, (pg, ) = _grads(g_loss)
        grad, skip = _unit_grad(ctx, (), lambda: torch.empty(B, N + 1, dtype=torch.float32, device=g.device))
        with on_device(g.device):
            rc = lib().b200rl_fqf_fraction_bwd(ptr(g), pg, B, N, skip, ptr(grad), stream_ptr())
        _lib.check(rc, 'b200rl_fqf_fraction_bwd')
        return (None, None, grad) + (None, ) * 6


# ----------------------------------------------------------------------------------------------------------------
# distributional n-step TD (C51)
# ----------------------------------------------------------------------------------------------------------------
class DistNStepTDFunction(torch.autograd.Function):
    """loss (differentiable w.r.t. dist) and the unweighted per-sample error; the forward launch also writes the gradient for
    a unit upstream gradient (verified on the device by the backward launch, as QNStepTDFunction)."""

    @staticmethod
    def forward(ctx, dist, next_n_dist, act, next_n_act, reward, done, weight, w_stride, value_gamma, vg_stride,
                support, B, A, N, n_atom, nstep, gamma, v_min, v_max, bad_flag):
        dev = dist.device
        R = B * A
        loss = torch.empty((), dtype=torch.float32, device=dev)
        td = torch.empty(R, dtype=torch.float32, device=dev)
        proj = torch.empty(R, n_atom, dtype=torch.float32, device=dev)
        grad_unit = torch.empty_like(dist) if ctx.needs_input_grad[0] else None
        with on_device(dev):
            ws = workspace(dev)
            rc = lib().b200rl_dntd_fwd(
                ptr(dist), ptr(next_n_dist), ptr(act), ptr(next_n_act), ptr(reward), ptr(done), ptr(weight), w_stride,
                ptr(value_gamma), vg_stride, ptr(support), B, A, N, n_atom, nstep, gamma, v_min, v_max, ptr(loss),
                ptr(td), ptr(proj), ptr(bad_flag), ptr(grad_unit), ptr(ws), ws.numel() * 4, stream_ptr()
            )
        _lib.check(rc, 'b200rl_dntd_fwd')
        ctx.save_for_backward(dist, act, proj, weight)
        ctx.cfg = (R, N, n_atom, w_stride)
        ctx.spec = grad_unit
        ctx.set_materialize_grads(False)
        return loss, td

    @staticmethod
    def backward(ctx, g_loss, g_td):
        if g_loss is None and g_td is None:
            return (None, ) * 20
        dist, act, proj, weight = ctx.saved_tensors
        R, N, n_atom, w_stride = ctx.cfg
        keep, (pg, ptd) = _grads(g_loss, g_td)
        grad, skip = _unit_grad(ctx, (g_td, ), lambda: torch.empty_like(dist))
        with on_device(dist.device):
            rc = lib().b200rl_dntd_bwd(
                ptr(dist), ptr(act), ptr(proj), ptr(weight), w_stride, pg, ptd, R, N, n_atom, skip, ptr(grad),
                stream_ptr()
            )
        _lib.check(rc, 'b200rl_dntd_bwd')
        return (grad, ) + (None, ) * 19


# ----------------------------------------------------------------------------------------------------------------
# lambda returns / TD(lambda)
# ----------------------------------------------------------------------------------------------------------------
def lambda_returns_(value, reward, gammas, gamma, lambdas, lambda_, done, upgo_mode):
    T, B = reward.shape
    ret = torch.empty_like(reward)
    with on_device(value.device):
        rc = lib().b200rl_lambda_returns(
            ptr(value), ptr(reward), ptr(gammas), float(gamma), ptr(lambdas), float(lambda_), ptr(done),
            1 if upgo_mode else 0, T, B, ptr(ret), stream_ptr()
        )
    _lib.check(rc, 'b200rl_lambda_returns')
    return ret


class LambdaReturnsFunction(torch.autograd.Function):
    """generalized_lambda_returns / upgo_returns with the reference's differentiability (td.py:1574-1651 is plain torch
    arithmetic): gradients reach bootstrap_values, rewards and -- when they are tensors that require grad -- gammas and
    lambda_.  Backward is the transposed scan (csrc/td.cu: lambda_returns_bwd_kernel), one launch."""

    @staticmethod
    def forward(ctx, value, reward, gammas, lambdas, done, gamma, lambda_, upgo_mode):
        ret = lambda_returns_(value, reward, gammas, gamma, lambdas, lambda_, done, upgo_mode)
        ctx.save_for_backward(value, reward, gammas, lambdas, done, ret)
        ctx.scal = (float(gamma), float(lambda_), 1 if upgo_mode else 0)
        return ret

    @staticmethod
    def backward(ctx, g_ret):
        value, reward, gammas, lambdas, done, ret = ctx.saved_tensors
        gamma, lambda_, upgo = ctx.scal
        T, B = reward.shape
        g = f32c(g_ret)
        need = ctx.needs_input_grad
        gv = torch.empty_like(value)
        gr = torch.empty_like(reward) if need[1] else None
        gg = torch.empty_like(reward) if (need[2] and gammas is not None) else None
        gl = torch.empty_like(reward) if (need[3] and lambdas is not None) else None
        with on_device(value.device):
            rc = lib().b200rl_lambda_returns_bwd(
                ptr(g), ptr(value), ptr(reward), ptr(ret), ptr(gammas), gamma, ptr(lambdas), lambda_, ptr(done), upgo,
                T, B, ptr(gv), ptr(gr), ptr(gg), ptr(gl), stream_ptr()
            )
        _lib.check(rc, 'b200rl_lambda_returns_bwd')
        return gv if need[0] else None, gr, gg, gl, None, None, None, None


class TBCrossEntropyFunction(torch.autograd.Function):
    """tb_cross_entropy (upgo.py:7-43): ce (TB) = sum_k mask_k * log softmax(logit)[label]; gradient reaches ``logit``."""

    @staticmethod
    def forward(ctx, logit, label, mask, TB, K, N):
        ce = torch.empty(TB, dtype=torch.float32, device=logit.device)
        with on_device(logit.device):
            rc = lib().b200rl_tb_cross_entropy_fwd(ptr(logit), ptr(label), ptr(mask), TB, K, N, ptr(ce), stream_ptr())
        _lib.check(rc, 'b200rl_tb_cross_entropy_fwd')
        ctx.save_for_backward(logit, label, mask)
        ctx.cfg = (TB, K, N)
        return ce

    @staticmethod
    def backward(ctx, g_ce):
        logit, label, mask = ctx.saved_tensors
        TB, K, N = ctx.cfg
        g = f32c(g_ce).reshape(-1)
        grad = torch.empty_like(logit)
        with on_device(logit.device):
            rc = lib().b200rl_tb_cross_entropy_bwd(ptr(logit), ptr(label), ptr(mask), ptr(g), TB, K, N, ptr(grad),
                                                   stream_ptr())
        _lib.check(rc, 'b200rl_tb_cross_entropy_bwd')
        return grad, None, None, None, None, None


class _ScaleSaved(torch.autograd.Function):
    """loss whose gradient w.r.t. ``x`` was produced by the forward kernel for a unit upstream gradient."""

    @staticmethod
    def forward(ctx, x, loss, saved_grad):
        ctx.save_for_backward(saved_grad)
        return loss.view_as(loss)

    @staticmethod
    def backward(ctx, g):
        saved, = ctx.saved_tensors
        out = torch.empty_like(saved)
        keep, (pg, ) = _grads(g)
        with on_device(saved.device):
            rc = lib().b200rl_scale(pg, ptr(saved), ptr(out), saved.numel(), stream_ptr())
        _lib.check(rc, 'b200rl_scale')
        return out, None, None


def td_lambda_(value, reward, weight, gamma, lambda_):
    T, B = reward.shape
    dev = value.device
    loss = torch.empty((), dtype=torch.float32, device=dev)
    dvalue = torch.empty_like(value)
    with on_device(dev):
        ws = workspace(dev)
        rc = lib().b200rl_td_lambda_fwd(
            ptr(value), ptr(reward), ptr(weight), float(gamma), float(lambda_), T, B, ptr(loss), ptr(dvalue), ptr(ws),
            ws.numel() * 4, stream_ptr()
        )
    _lib.check(rc, 'b200rl_td_lambda_fwd')
    if value.requires_grad and torch.is_grad_enabled():
        return _ScaleSaved.apply(value, loss, dvalue)
    return loss


# ----------------------------------------------------------------------------------------------------------------
# UPGO head
# ----------------------------------------------------------------------------------------------------------------
class UPGOFunction(torch.autograd.Function):
    """upgo_loss head (upgo.py:77-111).  The forward launch also writes d loss / d logit for a unit upstream gradient while each
    row is still in L1 (ONE pass over the logits); backward verifies the upstream gradient on the device and recomputes only
    when it is not 1 (or on a repeated backward)."""

    @staticmethod
    def forward(ctx, logit, action, mask, rho, ret, value, TB, K, N):
        dev = logit.device
        loss = torch.empty((), dtype=torch.float32, device=dev)
        adv = torch.empty(TB, dtype=torch.float32, device=dev)
        grad_unit = torch.empty_like(logit) if ctx.needs_input_grad[0] else None
        with on_device(dev):
            ws = workspace(dev)
            rc = lib().b200rl_upgo_head_fwd(
                ptr(logit), ptr(action), ptr(mask), ptr(rho), ptr(ret), ptr(value), TB, K, N, ptr(loss), ptr(adv),
                ptr(grad_unit), ptr(ws), ws.numel() * 4, stream_ptr()
            )
        _lib.check(rc, 'b200rl_upgo_head_fwd')
        ctx.save_for_backward(logit, action, mask, adv)
        ctx.cfg = (TB, K, N)
        ctx.spec = grad_unit
        return loss

    @staticmethod
    def backward(ctx, g):
        logit, action, mask, adv = ctx.saved_tensors
        TB, K, N = ctx.cfg
        grad, skip = _unit_grad(ctx, (), lambda: torch.empty_like(logit))
        keep, (pg, ) = _grads(g)
        with on_device(logit.device):
            rc = lib().b200rl_upgo_head_bwd(
                ptr(logit), ptr(action), ptr(mask), ptr(adv), pg, TB, K, N, skip, ptr(grad), stream_ptr()
            )
        _lib.check(rc, 'b200rl_upgo_head_bwd')
        return (grad, ) + (None, ) * 8


class A2CFunction(torch.autograd.Function):
    """a2c_error (ding/rl_utils/a2c.py:10-44): three differentiable 0-dim losses; gradients reach logit and value.  One launch
    forward (losses + gradients for the expected upstream gradients), one verification launch backward (csrc/heads.cu)."""

    @staticmethod
    def forward(ctx, logit, value, action, adv, return_, weight, S, N):
        dev = logit.device
        out = torch.empty(4, dtype=torch.float32, device=dev)
        want = ctx.needs_input_grad[0] or ctx.needs_input_grad[1]
        gl = torch.empty_like(logit) if want else None
        gv = torch.empty_like(value) if want else None
        g_used = torch.empty(4, dtype=torch.float32, device=dev) if want else None
        ctx.hint = ppo_hint(dev, 'a2c')
        with on_device(dev):
            ws = workspace(dev)
            rc = lib().b200rl_a2c_fwd_grad(ptr(logit), ptr(action), ptr(value), ptr(adv), ptr(return_), ptr(weight), S, N,
                                           ptr(ctx.hint) if want else None, 0, None, None, None, ptr(g_used), None, ptr(out),
                                           ptr(gl), ptr(gv), ptr(ws), ws.numel() * 4, stream_ptr())
        _lib.check(rc, 'b200rl_a2c_fwd_grad')
        ctx.save_for_backward(logit, value, action, adv, return_, weight)
        ctx.cfg = (S, N)
        ctx.spec = (gl, gv, g_used) if want else None
        ctx.set_materialize_grads(False)
        return out[0], out[1], out[2]

    @staticmethod
    def backward(ctx, g_p, g_v, g_e):
        logit, value, action, adv, return_, weight = ctx.saved_tensors
        S, N = ctx.cfg
        keep, (pp, pv, pe) = _grads(g_p, g_v, g_e)
        gl, gv, g_used = _forward_grads(ctx) or (torch.empty_like(logit), torch.empty_like(value), None)
        with on_device(logit.device):
            ws = workspace(logit.device)
            rc = lib().b200rl_a2c_fwd_grad(ptr(logit), ptr(action), ptr(value), ptr(adv), ptr(return_), ptr(weight), S, N,
                                           None, 1, pp, pv, pe, ptr(g_used), ptr(ctx.hint), None, ptr(gl), ptr(gv), ptr(ws),
                                           ws.numel() * 4, stream_ptr())
        _lib.check(rc, 'b200rl_a2c_fwd_grad(verify)')
        return gl, gv, None, None, None, None, None, None


class A2CContinuousFunction(torch.autograd.Function):
    """a2c_error_continuous (ding/rl_utils/a2c.py:50-88): three differentiable 0-dim losses; gradients reach mu, sigma and
    value.  One launch forward (losses + gradients for the expected upstream gradients), one verification launch backward
    (csrc/heads.cu)."""

    @staticmethod
    def forward(ctx, mu, sigma, value, action, adv, return_, weight, S, D):
        dev = mu.device
        out = torch.empty(4, dtype=torch.float32, device=dev)
        want = any(ctx.needs_input_grad[:3])
        gm = torch.empty_like(mu) if want else None
        gs = torch.empty_like(sigma) if want else None
        gv = torch.empty_like(value) if want else None
        g_used = torch.empty(4, dtype=torch.float32, device=dev) if want else None
        ctx.hint = ppo_hint(dev, 'a2cc')
        with on_device(dev):
            ws = workspace(dev)
            rc = lib().b200rl_a2c_continuous_fwd_grad(
                ptr(mu), ptr(sigma), ptr(action), ptr(value), ptr(adv), ptr(return_), ptr(weight), S, D,
                ptr(ctx.hint) if want else None, 0, None, None, None, ptr(g_used), None, ptr(out), ptr(gm), ptr(gs), ptr(gv),
                ptr(ws), ws.numel() * 4, stream_ptr())
        _lib.check(rc, 'b200rl_a2c_continuous_fwd_grad')
        ctx.save_for_backward(mu, sigma, value, action, adv, return_, weight)
        ctx.cfg = (S, D)
        ctx.spec = (gm, gs, gv, g_used) if want else None
        ctx.set_materialize_grads(False)
        return out[0], out[1], out[2]

    @staticmethod
    def backward(ctx, g_p, g_v, g_e):
        mu, sigma, value, action, adv, return_, weight = ctx.saved_tensors
        S, D = ctx.cfg
        keep, (pp, pv, pe) = _grads(g_p, g_v, g_e)
        gm, gs, gv, g_used = _forward_grads(ctx) or (torch.empty_like(mu), torch.empty_like(sigma), torch.empty_like(value),
                                                     None)
        with on_device(mu.device):
            ws = workspace(mu.device)
            rc = lib().b200rl_a2c_continuous_fwd_grad(
                ptr(mu), ptr(sigma), ptr(action), ptr(value), ptr(adv), ptr(return_), ptr(weight), S, D, None, 1, pp, pv,
                pe, ptr(g_used), ptr(ctx.hint), None, ptr(gm), ptr(gs), ptr(gv), ptr(ws), ws.numel() * 4, stream_ptr())
        _lib.check(rc, 'b200rl_a2c_continuous_fwd_grad(verify)')
        return gm, gs, gv, None, None, None, None, None, None


class PPOContinuousFunction(torch.autograd.Function):
    """ppo_error_continuous (ding/rl_utils/ppo.py:278-374): gradients reach mu_new, sigma_new and value_new (csrc/heads.cu).
    ``hint_kind`` names the call site's expected-upstream-gradient record (a key of ``_HINT_INIT``)."""

    @staticmethod
    def forward(ctx, mu, sigma, value_new, mu_old, sigma_old, mu_pre, sigma_pre, action, value_old, adv, return_, weight, S,
                D, clip_ratio, use_value_clip, dual_clip, kl_type, hint_kind, factor=None):
        dev = mu.device
        ctx.factor = factor  # happo_error_continuous's per-sample factor (S,) or None; kept alive for the backward launch
        out = torch.empty(8, dtype=torch.float32, device=dev)
        want = any(ctx.needs_input_grad[:3])
        gm = torch.empty_like(mu) if want else None
        gs = torch.empty_like(sigma) if want else None
        gv = torch.empty_like(value_new) if want else None
        g_used = torch.empty(4, dtype=torch.float32, device=dev) if want else None
        ctx.hint = ppo_hint(dev, hint_kind)
        ctx.args = (ptr(factor), S, D, clip_ratio, use_value_clip, dual_clip, kl_type)
        with on_device(dev):
            ws = workspace(dev)
            rc = lib().b200rl_ppo_continuous_fwd_grad(
                ptr(mu), ptr(sigma), ptr(mu_old), ptr(sigma_old), ptr(mu_pre), ptr(sigma_pre), ptr(action), ptr(value_new),
                ptr(value_old), ptr(adv), ptr(return_), ptr(weight), *ctx.args, ptr(ctx.hint) if want else None, 0, None,
                None, None, None, ptr(g_used), None, ptr(out), ptr(gm), ptr(gs), ptr(gv), ptr(ws), ws.numel() * 4,
                stream_ptr())
        _lib.check(rc, 'b200rl_ppo_continuous_fwd_grad')
        ctx.save_for_backward(mu, sigma, value_new, mu_old, sigma_old, mu_pre, sigma_pre, action, value_old, adv, return_,
                              weight)
        ctx.spec = (gm, gs, gv, g_used) if want else None
        ctx.set_materialize_grads(False)
        ctx.mark_non_differentiable(out)
        return out[0], out[1], out[2], out[3], out

    @staticmethod
    def backward(ctx, g_p, g_v, g_e, g_k, _g_out):
        (mu, sigma, value_new, mu_old, sigma_old, mu_pre, sigma_pre, action, value_old, adv, return_,
         weight) = ctx.saved_tensors
        keep, (pp, pv, pe, pk) = _grads(g_p, g_v, g_e, g_k)
        gm, gs, gv, g_used = _forward_grads(ctx) or (torch.empty_like(mu), torch.empty_like(sigma),
                                                     torch.empty_like(value_new), None)
        with on_device(mu.device):
            ws = workspace(mu.device)
            rc = lib().b200rl_ppo_continuous_fwd_grad(
                ptr(mu), ptr(sigma), ptr(mu_old), ptr(sigma_old), ptr(mu_pre), ptr(sigma_pre), ptr(action), ptr(value_new),
                ptr(value_old), ptr(adv), ptr(return_), ptr(weight), *ctx.args, None, 1, pp, pv, pe, pk, ptr(g_used),
                ptr(ctx.hint), None, ptr(gm), ptr(gs), ptr(gv), ptr(ws), ws.numel() * 4, stream_ptr())
        _lib.check(rc, 'b200rl_ppo_continuous_fwd_grad(verify)')
        return (gm, gs, gv) + (None, ) * 17


class ImpalaMaskFunction(torch.autograd.Function):
    """IMPALAPolicy._reshape_data masking (ding/policy/impala.py:316-322): values (T+1, B) (differentiable), rewards, done
    (T, B) -> (values', rewards', weights).  The reference multiplies ``values[1:]`` in place, so gradient reaches the critic
    output through the mask; backward is the same kernel applied to the upstream gradient."""

    @staticmethod
    def forward(ctx, values, rewards, done):
        T, B = rewards.shape
        vo = torch.empty_like(values)
        ro = torch.empty_like(rewards)
        wo = torch.empty_like(rewards)
        with on_device(values.device):
            rc = lib().b200rl_impala_mask(ptr(values), ptr(rewards), ptr(done), T, B, ptr(vo), ptr(ro), ptr(wo), stream_ptr())
        _lib.check(rc, 'b200rl_impala_mask')
        ctx.save_for_backward(done)
        ctx.mark_non_differentiable(ro, wo)
        return vo, ro, wo

    @staticmethod
    def backward(ctx, g_v, _g_r, _g_w):
        done, = ctx.saved_tensors
        T, B = done.shape
        g = f32c(g_v)
        out = torch.empty_like(g)
        with on_device(g.device):
            rc = lib().b200rl_impala_mask(ptr(g), None, ptr(done), T, B, ptr(out), None, None, stream_ptr())
        _lib.check(rc, 'b200rl_impala_mask')
        return out, None, None


# ----------------------------------------------------------------------------------------------------------------
# V-trace
# ----------------------------------------------------------------------------------------------------------------
# True: the one-launch kernel (csrc/vtws.cu) also writes the gradients for the expected upstream gradients
# (``vtrace_hint``, IMPALA's loss weights to start with), verified by the backward pass.  False: rows / scan / backward
# kernels.
VTRACE_FUSED = True


class VTraceFunction(torch.autograd.Function):

    @staticmethod
    def forward(ctx, target_output, value, behaviour_output, action, reward, weight, gamma, lambda_, rho_clip, c_clip,
                rho_pg_clip):
        T, B = reward.shape
        N = target_output.shape[-1]
        dev = target_output.device
        out = torch.empty(4, dtype=torch.float32, device=dev)
        L = lib()
        tensors = (ptr(target_output), ptr(behaviour_output), ptr(action), ptr(value), ptr(reward), ptr(weight))
        want_grad = ctx.needs_input_grad[0] or ctx.needs_input_grad[1]
        ctx.cfg = (T, B, N)
        ctx.scal = None  # the scalars of the verify launch: set on the one-launch path only
        with on_device(dev):
            ws = workspace(dev)
            if VTRACE_FUSED:
                grad_logit = torch.empty_like(target_output) if want_grad else None
                grad_value = torch.empty(T + 1, B, dtype=torch.float32, device=dev) if want_grad else None
                if L.b200rl_vtrace_fused_supported(*tensors, T, B, N, ptr(grad_logit), ptr(grad_value)):
                    g_used = torch.empty(3, dtype=torch.float32, device=dev) if want_grad else None
                    rc = L.b200rl_vtrace_fwd_grad(
                        *tensors, T, B, N, gamma, lambda_, rho_clip, c_clip, rho_pg_clip,
                        ptr(vtrace_hint(dev)) if want_grad else None, 0, None, None, None, ptr(g_used), None, ptr(out),
                        ptr(grad_logit), ptr(grad_value), ptr(ws), ws.numel() * 4, stream_ptr()
                    )
                    _lib.check(rc, 'b200rl_vtrace_fwd_grad')
                    ctx.spec = (grad_logit, grad_value, g_used) if want_grad else None
                    ctx.scal = (gamma, lambda_, rho_clip, c_clip, rho_pg_clip)
                    ctx.save_for_backward(target_output, behaviour_output, action, value, reward, weight)
                    return out[0], out[1], out[2]
            lp = torch.empty(T, B, dtype=torch.float32, device=dev)
            cpg = torch.empty(T, B, dtype=torch.float32, device=dev)
            dv = torch.empty(T, B, dtype=torch.float32, device=dev)
            rc = L.b200rl_vtrace_fwd(
                *tensors, T, B, N, gamma, lambda_, rho_clip, c_clip, rho_pg_clip, ptr(out), ptr(lp), ptr(cpg), ptr(dv),
                ptr(ws), ws.numel() * 4, stream_ptr()
            )
        _lib.check(rc, 'b200rl_vtrace_fwd')
        ctx.save_for_backward(target_output, action, weight, cpg, dv)
        return out[0], out[1], out[2]

    @staticmethod
    def backward(ctx, g_p, g_v, g_e):
        T, B, N = ctx.cfg
        keep, (pp, pv, pe) = _grads(g_p, g_v, g_e)
        if ctx.scal is not None:
            target_output, behaviour_output, action, value, reward, weight = ctx.saved_tensors
            dev = target_output.device
            grad_logit, grad_value, g_used = _forward_grads(ctx) or (
                torch.empty_like(target_output), torch.empty(T + 1, B, dtype=torch.float32, device=dev), None)
            with on_device(dev):
                ws = workspace(dev)
                rc = lib().b200rl_vtrace_fwd_grad(
                    ptr(target_output), ptr(behaviour_output), ptr(action), ptr(value), ptr(reward), ptr(weight), T, B,
                    N, *ctx.scal, None, 1, pp, pv, pe, ptr(g_used), ptr(vtrace_hint(dev)), None, ptr(grad_logit),
                    ptr(grad_value), ptr(ws), ws.numel() * 4, stream_ptr()
                )
            _lib.check(rc, 'b200rl_vtrace_fwd_grad(verify)')
            return (grad_logit, grad_value) + (None, ) * 9
        target_output, action, weight, cpg, dv = ctx.saved_tensors
        dev = target_output.device
        grad_logit = torch.empty_like(target_output)
        grad_value = torch.empty(T + 1, B, dtype=torch.float32, device=dev)
        with on_device(dev):
            rc = lib().b200rl_vtrace_bwd(
                ptr(target_output), ptr(action), ptr(weight), ptr(cpg), ptr(dv), pp, pv, pe, T, B, N, ptr(grad_logit),
                ptr(grad_value), stream_ptr()
            )
        _lib.check(rc, 'b200rl_vtrace_bwd')
        return (grad_logit, grad_value) + (None, ) * 9


class VTraceContinuousFunction(torch.autograd.Function):
    """vtrace_error_continuous_action (ding/rl_utils/vtrace.py:139-212): rows kernel -> shared scan -> backward rows kernel."""

    @staticmethod
    def forward(ctx, mu, sigma, value, mu_b, sigma_b, action, reward, weight, D, gamma, lambda_, rho_clip, c_clip,
                rho_pg_clip):
        T, B = reward.shape
        dev = mu.device
        out = torch.empty(4, dtype=torch.float32, device=dev)
        lp = torch.empty(T, B, dtype=torch.float32, device=dev)
        cpg = torch.empty(T, B, dtype=torch.float32, device=dev)
        dv = torch.empty(T, B, dtype=torch.float32, device=dev)
        with on_device(dev):
            ws = workspace(dev)
            rc = lib().b200rl_vtrace_continuous_fwd(
                ptr(mu), ptr(sigma), ptr(mu_b), ptr(sigma_b), ptr(action), ptr(value), ptr(reward), ptr(weight), T, B, D,
                gamma, lambda_, rho_clip, c_clip, rho_pg_clip, ptr(out), ptr(lp), ptr(cpg), ptr(dv), ptr(ws),
                ws.numel() * 4, stream_ptr())
        _lib.check(rc, 'b200rl_vtrace_continuous_fwd')
        ctx.save_for_backward(mu, sigma, action, weight, cpg, dv)
        ctx.cfg = (T, B, D)
        ctx.set_materialize_grads(False)
        return out[0], out[1], out[2]

    @staticmethod
    def backward(ctx, g_p, g_v, g_e):
        mu, sigma, action, weight, cpg, dv = ctx.saved_tensors
        T, B, D = ctx.cfg
        keep, (pp, pv, pe) = _grads(g_p, g_v, g_e)
        gm, gs = torch.empty_like(mu), torch.empty_like(sigma)
        gv = torch.empty(T + 1, B, dtype=torch.float32, device=mu.device)
        with on_device(mu.device):
            rc = lib().b200rl_vtrace_continuous_bwd(ptr(mu), ptr(sigma), ptr(action), ptr(weight), ptr(cpg), ptr(dv), pp, pv,
                                                    pe, T, B, D, ptr(gm), ptr(gs), ptr(gv), stream_ptr())
        _lib.check(rc, 'b200rl_vtrace_continuous_bwd')
        return (gm, gs, gv) + (None, ) * 11


# ----------------------------------------------------------------------------------------------------------------
# language-model policy losses on vocabulary-scale logits (csrc/vocab.cu)
# ----------------------------------------------------------------------------------------------------------------
_LOGIT_DTYPES = {torch.float32: 0, torch.bfloat16: 1}  # B200RL_DTYPE_F32, B200RL_DTYPE_BF16


def logit_dtype(*logits):
    """dtype code of csrc/vocab.cu for the logits of one call: fp32 or bf16, every logit tensor in the same dtype.  These
    kernels read bf16 as it arrives and compute in fp32; every other operator keeps to ``f32c``."""
    dt = logits[0].dtype
    if dt not in _LOGIT_DTYPES:
        raise TypeError("di_engine_b200: logits must be float32 or bfloat16 (got %s)" % dt)
    for t in logits[1:]:
        if t.dtype != dt:
            raise TypeError("di_engine_b200: all logits of one call must share a dtype (got %s and %s)" % (dt, t.dtype))
    return _LOGIT_DTYPES[dt]


def logits_c(t):
    """contiguous and 16-byte aligned, as the kernel's vector loads need (a view at an odd offset is copied)"""
    t = t.contiguous()
    return t if t.data_ptr() % 16 == 0 else t.clone()


class GRPOFunction(torch.autograd.Function):
    """grpo_policy_error (ding/rl_utils/grpo.py) on logits (B, S, V): outputs loss (differentiable w.r.t. logit_new),
    approx_kl and clipfrac.  ONE forward launch (+ the loss-sum finalize) also writes d loss / d logit_new for a unit
    upstream gradient; ``backward`` hands that buffer to autograd after a launch that returns at once on the device when
    the upstream gradient really is 1, and recomputes otherwise from the saved per-row logsumexp and coefficient."""

    @staticmethod
    def forward(ctx, logit_new, logit_old, logit_ref, action, adv, weight, dt, clip_ratio, beta):
        B, S, V = logit_new.shape
        out, lse, dlp, grad = _vocab_outputs(ctx, logit_new)
        with on_device(logit_new.device):
            ws = workspace(logit_new.device)
            rc = lib().b200rl_grpo_fwd_grad(dt, ptr(logit_new), ptr(logit_old), ptr(logit_ref), ptr(action), ptr(adv),
                                            ptr(weight), B, S, V, clip_ratio, beta, ptr(out), ptr(lse), ptr(dlp),
                                            ptr(grad), ptr(ws), ws.numel() * 4, stream_ptr())
        _lib.check(rc, 'b200rl_grpo_fwd_grad')
        return _vocab_saved(ctx, logit_new, action, lse, dlp, grad, dt, out)

    @staticmethod
    def backward(ctx, g_loss, _g_kl, _g_cf):
        return (_vocab_backward(ctx, g_loss), ) + (None, ) * 8


class RLOOFunction(torch.autograd.Function):
    """rloo_policy_error (ding/rl_utils/rloo.py) on logits (B, S, V); the leave-one-out advantage is formed in the kernel
    from reward (K, B / K).  Outputs and backward as ``GRPOFunction``."""

    @staticmethod
    def forward(ctx, logit_new, logit_old, action, reward, weight, dt, clip_ratio):
        B, S, V = logit_new.shape
        out, lse, dlp, grad = _vocab_outputs(ctx, logit_new)
        with on_device(logit_new.device):
            ws = workspace(logit_new.device)
            rc = lib().b200rl_rloo_fwd_grad(dt, ptr(logit_new), ptr(logit_old), ptr(action), ptr(reward), reward.shape[0],
                                            ptr(weight), B, S, V, clip_ratio, ptr(out), ptr(lse), ptr(dlp), ptr(grad),
                                            ptr(ws), ws.numel() * 4, stream_ptr())
        _lib.check(rc, 'b200rl_rloo_fwd_grad')
        return _vocab_saved(ctx, logit_new, action, lse, dlp, grad, dt, out)

    @staticmethod
    def backward(ctx, g_loss, _g_kl, _g_cf):
        return (_vocab_backward(ctx, g_loss), ) + (None, ) * 6


class PPOLMFunction(torch.autograd.Function):
    """ppo_policy_error (ding/rl_utils/ppo.py:143-230) on token rows: logits (..., V) fp32 or bf16, action / adv / weight
    over the same rows.  Outputs: policy_loss, entropy_loss, kl_div (differentiable; the gradient reaches logit_new only)
    and the raw result vector {policy, entropy, kl, approx_kl, clipfrac} (non differentiable).  The forward launch also
    writes d / d logit_new for the upstream gradients the call site's record ``hint_kind`` expects (its policy, entropy and
    kl slots); ``backward`` hands that buffer to autograd after a launch that returns at once on the device when the
    expectation held, and otherwise recomputes from the saved per-row values -- PPOFunction's scheme, at vocabulary scale."""

    @staticmethod
    def forward(ctx, logit_new, logit_old, logit_pre, action, adv, weight, dt, clip_ratio, dual_clip, kl_type, entropy,
                hint_kind):
        dev = logit_new.device
        V = logit_new.shape[-1]
        rows = logit_new.numel() // V
        out = torch.empty(5, dtype=torch.float32, device=dev)
        lse = torch.empty(rows, dtype=torch.float32, device=dev)
        ent = torch.empty(rows, dtype=torch.float32, device=dev) if entropy else None
        dpol = torch.empty(rows, dtype=torch.float32, device=dev)
        dkl = torch.empty(rows, dtype=torch.float32, device=dev) if logit_pre is not None else None
        want = ctx.needs_input_grad[0]
        grad = torch.empty_like(logit_new) if want else None
        g_used = torch.empty(4, dtype=torch.float32, device=dev) if want else None
        ctx.hint_kind = hint_kind
        with on_device(dev):
            ws = workspace(dev)
            rc = lib().b200rl_ppo_lm_fwd_grad(
                dt, ptr(logit_new), ptr(logit_old), ptr(logit_pre), ptr(action), ptr(adv), ptr(weight), rows, V,
                clip_ratio, dual_clip, kl_type, 1 if entropy else 0, ptr(ppo_hint(dev, hint_kind)) if want else None,
                ptr(g_used), ptr(out), ptr(lse), ptr(ent), ptr(dpol), ptr(dkl), ptr(grad), ptr(ws), ws.numel() * 4,
                stream_ptr())
        _lib.check(rc, 'b200rl_ppo_lm_fwd_grad')
        ctx.save_for_backward(logit_new, action, weight, lse, ent, dpol, dkl)
        ctx.dt = dt
        ctx.spec = (grad, g_used) if want else None
        ctx.mark_non_differentiable(out)
        return out[0], out[1], out[2], out

    @staticmethod
    def backward(ctx, g_p, g_e, g_k, _g_out):
        logit_new, action, weight, lse, ent, dpol, dkl = ctx.saved_tensors
        dev = logit_new.device
        keep, (pp, pe, pk) = _grads(g_p, g_e, g_k)
        spec = _forward_grads(ctx)
        if spec is not None:  # valid if the expectation held; the kernel checks on the device
            grad, g_used = spec
            p_used, p_hint = ptr(g_used), ptr(ppo_hint(dev, ctx.hint_kind))
        else:  # a repeated backward: null g_used / hint -> the kernel recomputes
            grad, p_used, p_hint = torch.empty_like(logit_new), None, None
        V = logit_new.shape[-1]
        with on_device(dev):
            rc = lib().b200rl_ppo_lm_bwd(ctx.dt, ptr(logit_new), ptr(action), ptr(weight), lse.numel(), V, ptr(lse),
                                         ptr(ent), ptr(dpol), ptr(dkl), pp, pe, pk, p_used, p_hint, ptr(grad),
                                         stream_ptr())
        _lib.check(rc, 'b200rl_ppo_lm_bwd')
        return (grad, ) + (None, ) * 11


class A2CLMFunction(torch.autograd.Function):
    """a2c_error (ding/rl_utils/a2c.py:10-44) on token rows: logit (..., V) fp32 or bf16; value, action, adv, return_,
    weight over the same rows, value fp32.  Outputs policy_loss, value_loss, entropy_loss (differentiable; the gradient
    reaches logit and value).  The forward launch also writes d / d logit and d / d value for the upstream gradients the
    ``'a2c'`` record expects; ``backward`` hands them to autograd after a launch that returns at once on the device when
    the expectation held, rewrites only d / d value when just the value weight changed, and otherwise recomputes from the
    saved per-row values -- A2CFunction's scheme, at vocabulary scale."""

    @staticmethod
    def forward(ctx, logit, value, action, adv, return_, weight, dt):
        dev = logit.device
        V = logit.shape[-1]
        rows = logit.numel() // V
        out = torch.empty(3, dtype=torch.float32, device=dev)
        lse, ent, dpol, dval = torch.empty(4, rows, dtype=torch.float32, device=dev).unbind(0)
        want = ctx.needs_input_grad[0] or ctx.needs_input_grad[1]
        gl = torch.empty_like(logit) if want else None
        gv = torch.empty_like(value) if want else None
        g_used = torch.empty(4, dtype=torch.float32, device=dev) if want else None
        with on_device(dev):
            ws = workspace(dev)
            rc = lib().b200rl_a2c_lm_fwd_grad(
                dt, ptr(logit), ptr(action), ptr(value), ptr(adv), ptr(return_), ptr(weight), rows, V,
                ptr(ppo_hint(dev, 'a2c')) if want else None, ptr(g_used), ptr(out), ptr(lse), ptr(ent), ptr(dpol),
                ptr(dval), ptr(gl), ptr(gv), ptr(ws), ws.numel() * 4, stream_ptr())
        _lib.check(rc, 'b200rl_a2c_lm_fwd_grad')
        ctx.save_for_backward(logit, value, action, weight, lse, ent, dpol, dval)
        ctx.dt = dt
        ctx.spec = (gl, gv, g_used) if want else None
        ctx.set_materialize_grads(False)
        return out[0], out[1], out[2]

    @staticmethod
    def backward(ctx, g_p, g_v, g_e):
        logit, value, action, weight, lse, ent, dpol, dval = ctx.saved_tensors
        dev = logit.device
        keep, (pp, pv, pe) = _grads(g_p, g_v, g_e)
        spec = _forward_grads(ctx)
        if spec is not None:  # valid if the expectation held; the kernel checks on the device
            gl, gv, g_used = spec
            p_used, p_hint = ptr(g_used), ptr(ppo_hint(dev, 'a2c'))
        else:  # a repeated backward: null g_used / hint -> the kernel recomputes
            gl, gv, p_used, p_hint = torch.empty_like(logit), torch.empty_like(value), None, None
        with on_device(dev):
            rc = lib().b200rl_a2c_lm_bwd(ctx.dt, ptr(logit), ptr(action), ptr(weight), lse.numel(), logit.shape[-1],
                                         ptr(lse), ptr(ent), ptr(dpol), ptr(dval), pp, pv, pe, p_used, p_hint, ptr(gl),
                                         ptr(gv), stream_ptr())
        _lib.check(rc, 'b200rl_a2c_lm_bwd')
        return gl, gv, None, None, None, None, None


def _vocab_outputs(ctx, logit_new):
    dev = logit_new.device
    rows = logit_new.shape[0] * logit_new.shape[1]
    out = torch.empty(3, dtype=torch.float32, device=dev)
    lse = torch.empty(rows, dtype=torch.float32, device=dev)
    dlp = torch.empty(rows, dtype=torch.float32, device=dev)
    grad = torch.empty_like(logit_new) if ctx.needs_input_grad[0] else None
    return out, lse, dlp, grad


def _vocab_saved(ctx, logit_new, action, lse, dlp, grad, dt, out):
    ctx.save_for_backward(logit_new, action, lse, dlp)
    ctx.dt = dt
    ctx.spec = grad
    ctx.set_materialize_grads(False)
    loss, approx_kl, clipfrac = out[0], out[1], out[2]
    ctx.mark_non_differentiable(approx_kl, clipfrac)
    return loss, approx_kl, clipfrac


def _vocab_backward(ctx, g_loss):
    if g_loss is None:
        return None
    logit_new, action, lse, dlp = ctx.saved_tensors
    keep, (pg, ) = _grads(g_loss)
    grad, skip = _unit_grad(ctx, (), lambda: torch.empty_like(logit_new))
    with on_device(logit_new.device):
        rc = lib().b200rl_token_logp_bwd(ctx.dt, ptr(logit_new), ptr(action), ptr(lse), ptr(dlp), pg, skip, lse.numel(),
                                         logit_new.shape[-1], ptr(grad), stream_ptr())
    _lib.check(rc, 'b200rl_token_logp_bwd')
    return grad


class TokenLogProbFunction(torch.autograd.Function):
    """log p(index) under softmax(logits) per token (ding/rl_utils/log_prob_utils.py): logits (rows, V) fp32 or bf16,
    index (rows) -> fp32 (rows).  Backward: d / d logits = g * (onehot - softmax), one launch."""

    @staticmethod
    def forward(ctx, logits, index, dt):
        rows, V = logits.shape
        lp = torch.empty(rows, dtype=torch.float32, device=logits.device)
        lse = torch.empty(rows, dtype=torch.float32, device=logits.device)
        with on_device(logits.device):
            rc = lib().b200rl_token_logp_fwd(dt, ptr(logits), ptr(index), rows, V, ptr(lp), ptr(lse), stream_ptr())
        _lib.check(rc, 'b200rl_token_logp_fwd')
        ctx.save_for_backward(logits, index, lse)
        ctx.dt = dt
        return lp

    @staticmethod
    def backward(ctx, g):
        logits, index, lse = ctx.saved_tensors
        g = g.float().contiguous()
        grad = torch.empty_like(logits)
        with on_device(logits.device):
            rc = lib().b200rl_token_logp_bwd(ctx.dt, ptr(logits), ptr(index), ptr(lse), ptr(g), None, 0, lse.numel(),
                                             logits.shape[-1], ptr(grad), stream_ptr())
        _lib.check(rc, 'b200rl_token_logp_bwd')
        return grad, None, None


def token_head_(lp_new, lp_old, lp_ref, adv, reward, weight, clip_ratio, beta):
    """The GRPO (``lp_ref`` given) or RLOO head on per-token log-probabilities (B, S) fp32 from a caller's own
    log_prob_fn: returns (loss, approx_kl, clipfrac); the gradient reaches ``lp_new`` (b200rl_scale of the saved
    unit-upstream gradient), and through it whatever computed it."""
    dev = lp_new.device
    B, S = lp_new.shape
    out = torch.empty(3, dtype=torch.float32, device=dev)
    dlp = torch.empty(B, S, dtype=torch.float32, device=dev)
    with on_device(dev):
        ws = workspace(dev)
        rc = lib().b200rl_token_head_fwd(ptr(lp_new), ptr(lp_old), ptr(lp_ref), ptr(adv), ptr(reward),
                                         0 if reward is None else reward.shape[0], ptr(weight), B, S, clip_ratio, beta,
                                         ptr(out), ptr(dlp), ptr(ws), ws.numel() * 4, stream_ptr())
    _lib.check(rc, 'b200rl_token_head_fwd')
    loss = out[0]
    if lp_new.requires_grad and torch.is_grad_enabled():
        loss = _ScaleSaved.apply(lp_new, loss, dlp)
    return loss, out[1], out[2]
