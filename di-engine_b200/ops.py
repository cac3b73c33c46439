"""Tensor-level operators over the C ABI (``include/b200rl.h``): allocation of outputs, stream / workspace plumbing and
``torch.autograd.Function`` wrappers.  torch is used for device memory, streams and autograd bookkeeping only; every
arithmetic step of the hot path runs in the CUDA kernels of ``csrc/``.

Nothing here computes on the CPU.  Host (CPU) tensors are accepted by the public API in ``rl_utils`` by staging them
to the current CUDA device and returning results on the host -- the "host buffers" end-to-end path.
"""
import os
import threading

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
    if not torch.compiler.is_compiling():  # a traced call loads the library when its custom ops run
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


def lasting(make, device):
    """``make()``, for a buffer kept for the life of the process (the workspace, the upstream-gradient records, cached
    constants).  CUDA graphs must not own such a buffer: torch.compile's ``mode="reduce-overhead"`` sends every allocation
    of its warm-up run to the graphs' private memory pool, whose blocks it hands out again to later graphs.  So the buffer is
    made on a helper thread, whose allocations go to the ordinary pool, and synchronised before it is used.  Inside a stream
    capture nothing may be allocated or synchronised, so a first use there is an error."""
    if device.type != 'cuda':
        return make()
    if torch.cuda.is_current_stream_capturing():
        raise _lib.B200RLError(
            "di_engine_b200: a workspace or upstream-gradient record is first needed inside a CUDA graph capture. Run the "
            "step once on the capturing stream before capturing it (torch.compile's mode='reduce-overhead' does so in its "
            "warm-up call; with torch.cuda.graph, run one eager step on the capture stream first)."
        )
    made = []

    def run():
        try:
            with torch.cuda.device(device):
                made.append(make())
                torch.cuda.current_stream().synchronize()
        except BaseException as e:  # re-raised on the calling thread
            made.append(e)

    t = threading.Thread(target=run)
    t.start()
    t.join()
    if isinstance(made[0], BaseException):
        raise made[0]
    return made[0]


def workspace(device):
    """One zero-initialised scratch buffer per (device, stream): launches sharing it are stream-ordered."""
    idx = device.index
    if idx is None:
        idx = torch.cuda.current_device() if device.type == 'cuda' else -1
    key = (idx, stream_ptr())
    ws = _WS.get(key)
    if ws is None:
        nbytes = lib().b200rl_workspace_bytes()
        ws = lasting(lambda: torch.zeros(nbytes // 4, dtype=torch.float32, device=device), device)
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
        t = lasting(lambda: torch.full((1, ), float(value), dtype=torch.float32, device=device), device)
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
    'coma': [0.001, 1.0, -0.01, 0.0],  # COMAPolicy: policy_weight, value_weight, -entropy_weight (policy/coma.py:77-81, 213-214)
}
_HINT = {}


def head_hint(device, kind, init):
    """device-resident expectation of the upstream gradients of a loss head (one record per head kind and device)"""
    key = (device.index, kind)
    h = _HINT.get(key)
    if h is None:
        h = lasting(lambda: torch.tensor(init, dtype=torch.float32, device=device), device)
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


# the value_norm modes of PPOFPolicy (ding/policy/ppof.py:167), in the order of b200rl_gae_returns_norm's argument
VALUE_NORMS = ('baseline', 'value_rescale', 'symlog', 'popart')
GAE_SEQ_MAX_T = 24576  # longest sequence csrc/policy.cu's one-launch kernel takes (GS_MAX_T)


def gae_returns_norm_(value, next_value, reward, done, traj_flag, gamma, lambda_, value_norm, std, mu, sigma, want_stats):
    """PPOFPolicy's advantage recompute (ding/policy/ppof.py:160-210) -- csrc/policy.cu.  value / next_value / reward /
    done / traj_flag (T, C) contiguous fp32 on one CUDA device; mu / sigma one device float each ('popart').
    -> (adv, value_out, return_out, stats3 or None, adv_stats2)."""
    T = value.shape[0]
    C = value.numel() // T
    dev = value.device
    adv = torch.empty_like(value)
    vout = torch.empty_like(value)
    rout = torch.empty_like(value)
    stats = torch.empty(3, dtype=torch.float32, device=dev) if want_stats else None
    astats = torch.empty(2, dtype=torch.float32, device=dev)
    scratch = None
    if not (C == 1 and T <= GAE_SEQ_MAX_T) and value_norm != 'baseline':  # the decode pass of the multi-launch path
        scratch = torch.empty((1 if value_norm == 'popart' else 2) * value.numel(), dtype=torch.float32, device=dev)
    with on_device(dev):
        ws = workspace(dev)
        rc = lib().b200rl_gae_returns_norm(
            ptr(value), ptr(next_value), ptr(reward), ptr(done), ptr(traj_flag), T, C, float(gamma), float(lambda_),
            VALUE_NORMS.index(value_norm), float(std), ptr(mu), ptr(sigma), ptr(adv), ptr(vout), ptr(rout), ptr(stats),
            ptr(astats), ptr(scratch), ptr(ws), ws.numel() * 4, stream_ptr()
        )
    _lib.check(rc, 'b200rl_gae_returns_norm')
    return adv, vout, rout, stats, astats


def value_map_fwd_(x, mode):
    """The forward launch of symlog / inv_symlog (ValueMapFunction and the ``b200rl::value_map`` custom op)."""
    y = torch.empty_like(x)
    if x.numel():
        with on_device(x.device):
            rc = lib().b200rl_value_map_fwd(mode, ptr(x), x.numel(), ptr(y), stream_ptr())
        _lib.check(rc, 'b200rl_value_map_fwd')
    return y


def value_map_bwd_(x, g, mode):
    """The backward launch of symlog / inv_symlog: d / d x for the contiguous fp32 upstream gradient ``g``."""
    dx = torch.empty_like(x)
    if x.numel():
        with on_device(x.device):
            rc = lib().b200rl_value_map_bwd(mode, ptr(x), ptr(g), x.numel(), ptr(dx), stream_ptr())
        _lib.check(rc, 'b200rl_value_map_bwd')
    return dx


class ValueMapFunction(torch.autograd.Function):
    """symlog (mode 0) / inv_symlog (mode 1) of ding/rl_utils/value_rescale.py:37-66 on a contiguous fp32 CUDA tensor; the
    backward is torch's autograd of the reference expression (include/b200rl.h)."""

    @staticmethod
    def forward(ctx, x, mode):
        y = value_map_fwd_(x, mode)
        ctx.mode = mode
        ctx.save_for_backward(x)
        return y

    @staticmethod
    def backward(ctx, g):
        x, = ctx.saved_tensors
        return value_map_bwd_(x, f32c(g, 'grad'), ctx.mode), None


# ----------------------------------------------------------------------------------------------------------------
# ppo
# ----------------------------------------------------------------------------------------------------------------
# True: the forward pass also writes the gradients for the expected upstream gradients (``ppo_hint``), verified by the
# backward pass.  False: separate backward kernel always.
PPO_FUSED_BACKWARD = True


def ppo_fwd_(logit_new, value_new, logit_old, action, value_old, adv, return_, weight, logit_pre, S, G, N, clip_ratio,
             use_value_clip, dual_clip, kl_type, hint_kind, adv_stats, factor, want_grad):
    """The forward launch of ppo_error (PPOFunction and the ``b200rl::ppo_loss`` custom op).  -> (the 8-float result vector,
    the forward-written (grad_logit, grad_value, g_used) or None when this launch wrote no gradients)."""
    dev = logit_new.device
    out = torch.empty(8, dtype=torch.float32, device=dev)
    L = lib()
    tensors = (ptr(logit_new), ptr(logit_old), ptr(logit_pre), ptr(action), ptr(value_new), ptr(value_old),
               ptr(adv), ptr(return_), ptr(weight))
    cfg = (S, G, N, clip_ratio, use_value_clip, dual_clip, kl_type, ptr(adv_stats), ptr(factor))
    spec = None
    with on_device(dev):
        ws = workspace(dev)
        if PPO_FUSED_BACKWARD and want_grad:
            grad_logit = torch.empty_like(logit_new)
            grad_value = torch.empty_like(value_new)
            if L.b200rl_ppo_fused_supported(*tensors, ptr(grad_logit), G, N):
                g_used = torch.empty(4, dtype=torch.float32, device=dev)
                rc = L.b200rl_ppo_fwd_grad(*tensors, *cfg, ptr(ppo_hint(dev, hint_kind)), ptr(g_used), ptr(out),
                                           ptr(grad_logit), ptr(grad_value), ptr(ws), ws.numel() * 4,
                                           stream_ptr())
                _lib.check(rc, 'b200rl_ppo_fwd_grad')
                spec = (grad_logit, grad_value, g_used)
        if spec is None:
            rc = L.b200rl_ppo_fwd(*tensors, *cfg, ptr(out), ptr(ws), ws.numel() * 4, stream_ptr())
            _lib.check(rc, 'b200rl_ppo_fwd')
    return out, spec


def ppo_bwd_(saved, cfg, upstream, spec, hint_kind):
    """The backward launch of ppo_error: ``saved`` the nine tensors of ppo_fwd_'s launch, ``cfg`` its (S, G, N, clip_ratio,
    use_value_clip, dual_clip, kl_type, adv_stats ptr, factor ptr), ``upstream`` the four device pointers of the upstream
    gradients (None = 0).  With ``spec`` (the forward-written gradients) it verifies them on the device and recomputes them
    in place on a mismatch; without, it computes into fresh buffers.  -> (grad_logit, grad_value)."""
    logit_new, value_new, logit_old, action, value_old, adv, return_, weight, logit_pre = saved
    dev = logit_new.device
    if spec is not None:  # valid if the expectation held; the kernel checks on the device
        grad_logit, grad_value, g_used = spec
        p_used, p_hint = ptr(g_used), ptr(ppo_hint(dev, hint_kind))
    else:  # no fused forward, or a repeated backward: null g_used / hint -> the kernel recomputes
        grad_logit = torch.empty_like(logit_new)
        grad_value = torch.empty_like(value_new)
        p_used, p_hint = None, None
    with on_device(dev):
        rc = lib().b200rl_ppo_bwd(
            ptr(logit_new), ptr(logit_old), ptr(logit_pre), ptr(action), ptr(value_new), ptr(value_old), ptr(adv),
            ptr(return_), ptr(weight), *cfg, *upstream, p_used, p_hint, ptr(grad_logit), ptr(grad_value),
            stream_ptr()
        )
    _lib.check(rc, 'b200rl_ppo_bwd')
    return grad_logit, grad_value


class PPOFunction(torch.autograd.Function):
    """Outputs: policy_loss, value_loss, entropy_loss, kl_div (differentiable 0-dim) and the raw 8-float result vector
    (non differentiable; [4]=approx_kl, [5]=clipfrac)."""

    @staticmethod
    def forward(ctx, logit_new, value_new, logit_old, action, value_old, adv, return_, weight, logit_pre, S, G, N,
                clip_ratio, use_value_clip, dual_clip, kl_type, hint_kind, adv_stats=None, factor=None):
        ctx.hint_kind = hint_kind
        ctx.adv_stats = adv_stats  # {mean, std + 1e-8} device floats or None; kept alive for the backward launch
        ctx.factor = factor        # happo_error's per-sample factor (S,) or None; likewise
        out, ctx.spec = ppo_fwd_(logit_new, value_new, logit_old, action, value_old, adv, return_, weight, logit_pre, S,
                                 G, N, clip_ratio, use_value_clip, dual_clip, kl_type, hint_kind, adv_stats, factor,
                                 ctx.needs_input_grad[0] or ctx.needs_input_grad[1])
        ctx.save_for_backward(logit_new, value_new, logit_old, action, value_old, adv, return_, weight, logit_pre)
        ctx.cfg = (S, G, N, clip_ratio, use_value_clip, dual_clip, kl_type, ptr(adv_stats), ptr(factor))
        ctx.mark_non_differentiable(out)
        p, v, e, k = out[0], out[1], out[2], out[3]
        return p, v, e, k, out

    @staticmethod
    def backward(ctx, g_p, g_v, g_e, g_k, _g_out):
        keep, upstream = _grads(g_p, g_v, g_e, g_k)
        grad_logit, grad_value = ppo_bwd_(ctx.saved_tensors, ctx.cfg, upstream, _forward_grads(ctx), ctx.hint_kind)
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


def ppo_value_fwd_(value_new, value_old, return_, weight, clip_ratio, use_value_clip, want_grad):
    """The one launch of ppo_value_error (ppo.py:233-275) -> (loss, d loss / d value_new for a unit upstream gradient, or
    None without ``want_grad``)"""
    dev = value_new.device
    loss = torch.empty((), dtype=torch.float32, device=dev)
    dvalue = torch.empty_like(value_new) if want_grad else None
    with on_device(dev):
        ws = workspace(dev)
        rc = lib().b200rl_ppo_value_fwd(
            ptr(value_new), ptr(value_old), ptr(return_), ptr(weight), value_new.numel(), float(clip_ratio),
            1 if use_value_clip else 0, ptr(loss), ptr(dvalue), ptr(ws), ws.numel() * 4, stream_ptr()
        )
    _lib.check(rc, 'b200rl_ppo_value_fwd')
    return loss, dvalue


def ppo_value_(value_new, value_old, return_, weight, clip_ratio, use_value_clip):
    """ppo_value_error (ppo.py:233-275): loss and, if needed, its gradient for a unit upstream gradient in one launch."""
    want_grad = value_new.requires_grad and torch.is_grad_enabled()
    loss, dvalue = ppo_value_fwd_(value_new, value_old, return_, weight, clip_ratio, use_value_clip, want_grad)
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
        loss, td, dcrit, target, prio, grad_unit = qntd_fwd_(
            q, next_n_q, action, next_n_action, reward, done, weight, value_gamma, vg_stride, gamma_ps, S, G, N, nstep,
            gamma, cum_reward, rescale, eps, criterion, crit_param, group_mean, seq_len, priority_mix, want_priority,
            ctx.needs_input_grad[0])
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
        qntd_bwd_(dcrit, weight, action, pg, ptd, S, G, N, group_mean, seq_len, skip, grad_q)
        return (grad_q.view(ctx.q_shape), ) + (None, ) * 23


def qntd_fwd_(q, next_n_q, action, next_n_action, reward, done, weight, value_gamma, vg_stride, gamma_ps, S, G, N, nstep,
              gamma, cum_reward, rescale, eps, criterion, crit_param, group_mean, seq_len, priority_mix, want_priority,
              want_grad):
    """The forward launch of the q-n-step TD family (QNStepTDFunction and the ``b200rl::qntd_fwd`` custom op).
    -> (loss, td, dcrit, target, prio or None, grad_unit or None)."""
    dev = q.device
    R = S * G
    loss = torch.empty((), dtype=torch.float32, device=dev)
    td = torch.empty(S if group_mean else R, dtype=torch.float32, device=dev)
    dcrit = torch.empty(R, dtype=torch.float32, device=dev)
    target = torch.empty(R, dtype=torch.float32, device=dev)
    prio = torch.empty(S // seq_len, dtype=torch.float32, device=dev) if want_priority else None
    grad_unit = torch.empty(R, N, dtype=torch.float32, device=dev) if want_grad else None
    with on_device(dev):
        ws = workspace(dev)
        rc = lib().b200rl_qntd_fwd(
            ptr(q), ptr(next_n_q), ptr(action), ptr(next_n_action), ptr(reward), ptr(done), ptr(weight),
            ptr(value_gamma), vg_stride, ptr(gamma_ps), S, G, N, nstep, gamma, cum_reward, rescale, eps, criterion,
            crit_param, group_mean, seq_len, priority_mix, ptr(loss), ptr(td), ptr(dcrit), ptr(target),
            ptr(grad_unit), ptr(prio), ptr(ws), ws.numel() * 4, stream_ptr()
        )
    _lib.check(rc, 'b200rl_qntd_fwd')
    return loss, td, dcrit, target, prio, grad_unit


def qntd_bwd_(dcrit, weight, action, pg, ptd, S, G, N, group_mean, seq_len, skip, grad_q):
    """The backward launch of the q-n-step TD family into ``grad_q``: ``pg`` / ``ptd`` the device pointers of the upstream
    gradients (None = 0); ``skip`` 1 when ``grad_q`` holds the forward-written unit gradient (verified on the device)."""
    with on_device(dcrit.device):
        rc = lib().b200rl_qntd_bwd(ptr(dcrit), ptr(weight), ptr(action), pg, ptd, S, G, N, group_mean, seq_len, skip,
                                   ptr(grad_q), stream_ptr())
    _lib.check(rc, 'b200rl_qntd_bwd')
    return grad_q


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
        loss, td, stats, saved, tn, t1, prio, grad_unit = dqfd_fwd_(
            q, next_n_q, next_q1, action, next_n_action, next_action1, reward, done, done1, weight, value_gamma,
            vg_stride, is_expert, S, N, nstep, gamma, cum_reward, rescale, eps, criterion, crit_param, lam_n, lam_1,
            lam_s, margin, seq_len, priority_mix, want_targets, want_priority, ctx.needs_input_grad[0])
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
        dqfd_bwd_(saved, weight, action, pg, ptd, (psn, ps1, psje), S, N, lam_n, lam_1, lam_s, seq_len, skip, grad_q)
        return (grad_q.view(ctx.q_shape), ) + (None, ) * (n_in - 1)


def dqfd_fwd_(q, next_n_q, next_q1, action, next_n_action, next_action1, reward, done, done1, weight, value_gamma,
              vg_stride, is_expert, S, N, nstep, gamma, cum_reward, rescale, eps, criterion, crit_param, lam_n, lam_1, lam_s,
              margin, seq_len, priority_mix, want_targets, want_priority, want_grad):
    """The forward launch of the DQfD family (DQfDTDFunction and the ``b200rl::dqfd_fwd`` custom op).
    -> (loss, td, stats (3,), saved (S, 4), tn or None, t1 or None, prio or None, grad_unit or None)."""
    dev = q.device
    loss = torch.empty((), dtype=torch.float32, device=dev)
    td = torch.empty(S, dtype=torch.float32, device=dev)
    stats = torch.empty(3, dtype=torch.float32, device=dev)
    saved = torch.empty(S, 4, dtype=torch.float32, device=dev)
    tn = torch.empty(S, dtype=torch.float32, device=dev) if want_targets else None
    t1 = torch.empty(S, dtype=torch.float32, device=dev) if want_targets else None
    prio = torch.empty(S // seq_len, dtype=torch.float32, device=dev) if want_priority else None
    grad_unit = torch.empty(S, N, dtype=torch.float32, device=dev) if want_grad else None
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
    return loss, td, stats, saved, tn, t1, prio, grad_unit


def dqfd_bwd_(saved, weight, action, pg, ptd, pstats, S, N, lam_n, lam_1, lam_s, seq_len, skip, grad_q):
    """The backward launch of the DQfD family into ``grad_q``: ``pg`` / ``ptd`` / ``pstats`` (three) the device pointers
    of the upstream gradients of loss, td and the statistics (None = 0); ``skip`` as qntd_bwd_."""
    with on_device(saved.device):
        rc = lib().b200rl_dqfd_bwd(ptr(saved), ptr(weight), ptr(action), pg, ptd, *pstats, S, N, lam_n, lam_1, lam_s,
                                   seq_len, skip, ptr(grad_q), stream_ptr())
    _lib.check(rc, 'b200rl_dqfd_bwd')
    return grad_q


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
        loss, td, dcrit, target, gap, clip, rec, grad_unit = soft_td_fwd_(
            q, target_q, next_q, action, reward, done, weight, value_gamma, vg_stride, mode, S, G, N, nstep, gamma, tau,
            alpha, cum_reward, criterion, crit_param, ctx.needs_input_grad[0])
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


def soft_td_fwd_(q, target_q, next_q, action, reward, done, weight, value_gamma, vg_stride, mode, S, G, N, nstep, gamma,
                 tau, alpha, cum_reward, criterion, crit_param, want_grad):
    """The forward launch of the soft TD losses (SoftTDFunction and the ``b200rl::soft_td_fwd`` custom op).
    -> (loss, td, dcrit, target, gap, clip, rec, grad_unit); the mode's missing statistics and grad_unit are None."""
    dev = q.device
    R = S * G
    loss = torch.empty((), dtype=torch.float32, device=dev)
    td = torch.empty(R, dtype=torch.float32, device=dev)
    dcrit = torch.empty(R, dtype=torch.float32, device=dev)
    target = torch.empty(R, dtype=torch.float32, device=dev)
    gap = torch.empty((), dtype=torch.float32, device=dev) if mode == 0 else None
    clip = torch.empty(R, dtype=torch.float32, device=dev) if mode == 0 else None
    rec = torch.empty(R, dtype=torch.float32, device=dev) if mode == 1 else None
    grad_unit = torch.empty(R, N, dtype=torch.float32, device=dev) if want_grad else None
    with on_device(dev):
        ws = workspace(dev)
        rc = lib().b200rl_soft_td_fwd(
            mode, ptr(q), ptr(target_q), ptr(next_q), ptr(action), ptr(reward), ptr(done), ptr(weight),
            ptr(value_gamma), vg_stride, S, G, N, nstep, gamma, tau, alpha, cum_reward, criterion, crit_param,
            ptr(loss), ptr(td), ptr(dcrit), ptr(target), ptr(grad_unit), ptr(gap), ptr(clip), ptr(rec), ptr(ws),
            ws.numel() * 4, stream_ptr()
        )
    _lib.check(rc, 'b200rl_soft_td_fwd')
    return loss, td, dcrit, target, gap, clip, rec, grad_unit


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
        loss, td, dtheta, grad_unit = quantile_fwd_(q, next_n_q, action, next_n_action, reward, done, tau, weight,
                                                    value_gamma, vg_stride, B, N, n_tau, n_tau_prime, nstep, gamma,
                                                    q_strides, nq_strides, tau_strides, form, kappa, ctx.needs_input_grad[0])
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
        return (quantile_bwd_(dtheta, weight, action, pg, ptd, B, N, n_tau, q_strides, skip, grad_q), ) + (None, ) * 20


def quantile_fwd_(q, next_n_q, action, next_n_action, reward, done, tau, weight, value_gamma, vg_stride, B, N, n_tau,
                  n_tau_prime, nstep, gamma, q_strides, nq_strides, tau_strides, form, kappa, want_grad):
    """The forward launch of the quantile TD family (QuantileTDFunction and the ``b200rl::quantile_fwd`` custom op).
    -> (loss, td, dtheta, grad_unit or None)."""
    dev = q.device
    loss = torch.empty((), dtype=torch.float32, device=dev)
    td = torch.empty(B, dtype=torch.float32, device=dev)
    dtheta = torch.empty(B, n_tau, dtype=torch.float32, device=dev)
    grad_unit = torch.empty_like(q) if want_grad else None
    with on_device(dev):
        ws = workspace(dev)
        rc = lib().b200rl_quantile_td_fwd(
            ptr(q), ptr(next_n_q), ptr(action), ptr(next_n_action), ptr(reward), ptr(done), ptr(tau), ptr(weight),
            ptr(value_gamma), vg_stride, B, N, n_tau, n_tau_prime, nstep, gamma, *q_strides, *nq_strides, *tau_strides,
            form, kappa, ptr(loss), ptr(td), ptr(dtheta), ptr(grad_unit), ptr(ws), ws.numel() * 4, stream_ptr()
        )
    _lib.check(rc, 'b200rl_quantile_td_fwd')
    return loss, td, dtheta, grad_unit


def quantile_bwd_(dtheta, weight, action, pg, ptd, B, N, n_tau, q_strides, skip, grad_q):
    """The backward launch of the quantile TD family into ``grad_q`` (``pg`` / ``ptd`` / ``skip`` as qntd_bwd_)."""
    with on_device(dtheta.device):
        rc = lib().b200rl_quantile_td_bwd(ptr(dtheta), ptr(weight), ptr(action), pg, ptd, B, N, n_tau, *q_strides, skip,
                                          ptr(grad_q), stream_ptr())
    _lib.check(rc, 'b200rl_quantile_td_bwd')
    return grad_q


class FQFFractionFunction(torch.autograd.Function):
    """FQF's fraction loss (td.py:1466-1513), differentiable w.r.t. ``quantiles`` only (q_tau_i and q_value enter detached,
    as the reference gathers them under no_grad); the forward launch also writes d loss / d quantiles for a unit upstream
    gradient (verified on the device by the backward launch, as QuantileTDFunction).  ``*_strides``: element strides of
    (sample, quantile[, action])."""

    @staticmethod
    def forward(ctx, q_tau_i, q_value, quantiles, action, B, N, qt_strides, qv_strides, qn_strides):
        loss, g, grad_unit = fqf_fraction_fwd_(q_tau_i, q_value, quantiles, action, B, N, qt_strides, qv_strides,
                                               qn_strides, ctx.needs_input_grad[2])
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
        return (None, None, fqf_fraction_bwd_(g, pg, B, N, skip, grad)) + (None, ) * 6


def fqf_fraction_fwd_(q_tau_i, q_value, quantiles, action, B, N, qt_strides, qv_strides, qn_strides, want_grad):
    """The forward launch of FQF's fraction loss (FQFFractionFunction and the ``b200rl::fqf_fraction_fwd`` custom op).
    -> (loss, g (B, N-1), grad_unit (B, N+1) or None)."""
    dev = quantiles.device
    loss = torch.empty((), dtype=torch.float32, device=dev)
    g = torch.empty(B, N - 1, dtype=torch.float32, device=dev)
    grad_unit = torch.empty(B, N + 1, dtype=torch.float32, device=dev) if want_grad else None
    with on_device(dev):
        ws = workspace(dev)
        rc = lib().b200rl_fqf_fraction_fwd(
            ptr(q_tau_i), ptr(q_value), ptr(quantiles), ptr(action), B, N, q_tau_i.shape[2], q_value.shape[2],
            *qt_strides, *qv_strides, *qn_strides, ptr(loss), ptr(g), ptr(grad_unit), ptr(ws), ws.numel() * 4,
            stream_ptr()
        )
    _lib.check(rc, 'b200rl_fqf_fraction_fwd')
    return loss, g, grad_unit


def fqf_fraction_bwd_(g, pg, B, N, skip, grad):
    """The backward launch of FQF's fraction loss into ``grad`` (B, N+1) (``pg`` / ``skip`` as qntd_bwd_)."""
    with on_device(g.device):
        rc = lib().b200rl_fqf_fraction_bwd(ptr(g), pg, B, N, skip, ptr(grad), stream_ptr())
    _lib.check(rc, 'b200rl_fqf_fraction_bwd')
    return grad


# ----------------------------------------------------------------------------------------------------------------
# distributional n-step TD (C51)
# ----------------------------------------------------------------------------------------------------------------
class DistNStepTDFunction(torch.autograd.Function):
    """loss (differentiable w.r.t. dist) and the unweighted per-sample error; the forward launch also writes the gradient for
    a unit upstream gradient (verified on the device by the backward launch, as QNStepTDFunction)."""

    @staticmethod
    def forward(ctx, dist, next_n_dist, act, next_n_act, reward, done, weight, w_stride, value_gamma, vg_stride,
                support, B, A, N, n_atom, nstep, gamma, v_min, v_max, bad_flag):
        loss, td, proj, grad_unit = dntd_fwd_(dist, next_n_dist, act, next_n_act, reward, done, weight, w_stride,
                                              value_gamma, vg_stride, support, B, A, N, n_atom, nstep, gamma, v_min,
                                              v_max, bad_flag, ctx.needs_input_grad[0])
        ctx.save_for_backward(dist, act, proj, weight)
        ctx.cfg = (B * A, N, n_atom, w_stride)
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
        dntd_bwd_(dist, act, proj, weight, w_stride, pg, ptd, R, N, n_atom, skip, grad)
        return (grad, ) + (None, ) * 19


def dntd_fwd_(dist, next_n_dist, act, next_n_act, reward, done, weight, w_stride, value_gamma, vg_stride, support, B, A, N,
              n_atom, nstep, gamma, v_min, v_max, bad_flag, want_grad):
    """The forward launch of dist_nstep_td_error (DistNStepTDFunction and the ``b200rl::dntd_fwd`` custom op).
    -> (loss, td, proj, grad_unit or None)."""
    dev = dist.device
    R = B * A
    loss = torch.empty((), dtype=torch.float32, device=dev)
    td = torch.empty(R, dtype=torch.float32, device=dev)
    proj = torch.empty(R, n_atom, dtype=torch.float32, device=dev)
    grad_unit = torch.empty_like(dist) if want_grad else None
    with on_device(dev):
        ws = workspace(dev)
        rc = lib().b200rl_dntd_fwd(
            ptr(dist), ptr(next_n_dist), ptr(act), ptr(next_n_act), ptr(reward), ptr(done), ptr(weight), w_stride,
            ptr(value_gamma), vg_stride, ptr(support), B, A, N, n_atom, nstep, gamma, v_min, v_max, ptr(loss),
            ptr(td), ptr(proj), ptr(bad_flag), ptr(grad_unit), ptr(ws), ws.numel() * 4, stream_ptr()
        )
    _lib.check(rc, 'b200rl_dntd_fwd')
    return loss, td, proj, grad_unit


def dntd_bwd_(dist, act, proj, weight, w_stride, pg, ptd, R, N, n_atom, skip, grad):
    """The backward launch of dist_nstep_td_error into ``grad`` (arguments as qntd_bwd_)."""
    with on_device(dist.device):
        rc = lib().b200rl_dntd_bwd(
            ptr(dist), ptr(act), ptr(proj), ptr(weight), w_stride, pg, ptd, R, N, n_atom, skip, ptr(grad),
            stream_ptr()
        )
    _lib.check(rc, 'b200rl_dntd_bwd')
    return grad


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
        keep, (pg, ) = _grads(g)
        return scale_(pg, saved), None, None


def scale_(pg, saved):
    """``*pg * saved`` into a fresh tensor: the backward launch of the heads whose forward saved the unit gradient."""
    out = torch.empty_like(saved)
    with on_device(saved.device):
        rc = lib().b200rl_scale(pg, ptr(saved), ptr(out), saved.numel(), stream_ptr())
    _lib.check(rc, 'b200rl_scale')
    return out


def td_lambda_fwd_(value, reward, weight, gamma, lambda_):
    """The one launch of td_lambda_error -> (loss, d loss / d value for a unit upstream gradient)."""
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
    return loss, dvalue


def td_lambda_(value, reward, weight, gamma, lambda_):
    loss, dvalue = td_lambda_fwd_(value, reward, weight, gamma, lambda_)
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
        loss, adv, grad_unit = upgo_fwd_(logit, action, mask, rho, ret, value, TB, K, N, ctx.needs_input_grad[0])
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
        return (upgo_bwd_(logit, action, mask, adv, pg, TB, K, N, skip, grad), ) + (None, ) * 8


def upgo_fwd_(logit, action, mask, rho, ret, value, TB, K, N, want_grad):
    """The forward launch of the upgo_loss head (UPGOFunction and the ``b200rl::upgo_fwd`` custom op).
    -> (loss, adv, grad_unit or None)."""
    dev = logit.device
    loss = torch.empty((), dtype=torch.float32, device=dev)
    adv = torch.empty(TB, dtype=torch.float32, device=dev)
    grad_unit = torch.empty_like(logit) if want_grad else None
    with on_device(dev):
        ws = workspace(dev)
        rc = lib().b200rl_upgo_head_fwd(
            ptr(logit), ptr(action), ptr(mask), ptr(rho), ptr(ret), ptr(value), TB, K, N, ptr(loss), ptr(adv),
            ptr(grad_unit), ptr(ws), ws.numel() * 4, stream_ptr()
        )
    _lib.check(rc, 'b200rl_upgo_head_fwd')
    return loss, adv, grad_unit


def upgo_bwd_(logit, action, mask, adv, pg, TB, K, N, skip, grad):
    """The backward launch of the upgo_loss head into ``grad`` (``pg`` / ``skip`` as qntd_bwd_)."""
    with on_device(logit.device):
        rc = lib().b200rl_upgo_head_bwd(
            ptr(logit), ptr(action), ptr(mask), ptr(adv), pg, TB, K, N, skip, ptr(grad), stream_ptr()
        )
    _lib.check(rc, 'b200rl_upgo_head_bwd')
    return grad


# ----------------------------------------------------------------------------------------------------------------
# COMA (coma.py:10-58): the value half on the lambda-return scan (td.cu, HEAD 2), the policy half on a row head (pg.cu)
# ----------------------------------------------------------------------------------------------------------------
def coma_fwd_(logit, q_value, target_q, action, reward, weight, T, B, A, N, gamma, lambda_, want_grad, want_dret):
    """The forward launch of coma_error (COMAFunction and the ``b200rl::coma_fwd`` custom op).
    -> (out (3,): policy, value, entropy loss; adv (T*B*A); dq ((T-1)*B*A); dret or None; (grad_logit, grad_q_value,
    g_used) or None)."""
    dev = logit.device
    out = torch.empty(3, dtype=torch.float32, device=dev)
    adv = torch.empty(T * B * A, dtype=torch.float32, device=dev)
    dq = torch.empty((T - 1) * B * A, dtype=torch.float32, device=dev)
    dret = torch.empty_like(dq) if want_dret else None
    spec = (torch.empty_like(logit), torch.empty_like(q_value),
            torch.empty(4, dtype=torch.float32, device=dev)) if want_grad else None
    with on_device(dev):
        ws = workspace(dev)
        gl, gq, g_used = spec if want_grad else (None, None, None)
        rc = lib().b200rl_coma_fwd(ptr(logit), ptr(q_value), ptr(target_q), ptr(action), ptr(reward), ptr(weight), T, B, A, N,
                                   float(gamma), float(lambda_), ptr(ppo_hint(dev, 'coma')) if want_grad else None,
                                   ptr(g_used), ptr(out), ptr(adv), ptr(dq), ptr(dret), ptr(gl), ptr(gq), ptr(ws),
                                   ws.numel() * 4, stream_ptr())
    _lib.check(rc, 'b200rl_coma_fwd')
    return out, adv, dq, dret, spec


def coma_bwd_(logit, action, weight, adv, dq, T, B, A, N, upstream, spec):
    """The verify launch of coma_error into ``spec`` = (grad_logit, grad_q_value, g_used) -- the forward-written buffers and
    their record, or fresh buffers and None (recompute).  ``upstream``: pointers of the policy, value and entropy gradients."""
    gl, gq, g_used = spec
    with on_device(logit.device):
        rc = lib().b200rl_coma_bwd(ptr(logit), ptr(action), ptr(weight), ptr(adv), ptr(dq), T, B, A, N, *upstream,
                                   ptr(g_used), ptr(ppo_hint(logit.device, 'coma')), ptr(gl), ptr(gq), stream_ptr())
    _lib.check(rc, 'b200rl_coma_bwd')
    return gl, gq


class COMAFunction(torch.autograd.Function):
    """coma_error's three differentiable 0-dim losses.  Gradients reach logit (policy and entropy terms) and q_value (the value
    loss, at the action column of rows t < T-1).  ``ret`` is None, or the differentiable lambda-return (T-1, B*A) that a
    caller builds when target_q_value / reward require grad: it receives d q_value_loss / d G (the returns themselves are
    recomputed in the kernel).  One forward launch pair writes the losses and the gradients for the ``'coma'`` record; one
    verify launch backward."""

    @staticmethod
    def forward(ctx, logit, q_value, target_q, action, reward, weight, ret, T, B, A, N, gamma, lambda_):
        want = ctx.needs_input_grad[0] or ctx.needs_input_grad[1]
        out, adv, dq, dret, spec = coma_fwd_(logit, q_value, target_q, action, reward, weight, T, B, A, N, gamma, lambda_,
                                             want, ret is not None)
        ctx.save_for_backward(logit, action, weight, adv, dq, dret)
        ctx.cfg = (T, B, A, N)
        ctx.spec = spec
        ctx.set_materialize_grads(False)
        return out[0], out[1], out[2]

    @staticmethod
    def backward(ctx, g_p, g_v, g_e):
        logit, action, weight, adv, dq, dret = ctx.saved_tensors
        T, B, A, N = ctx.cfg
        need = ctx.needs_input_grad
        keep, upstream = _grads(g_p, g_v, g_e)
        gl = gq = g_ret = None
        if need[0] or need[1]:
            spec = _forward_grads(ctx) or (torch.empty_like(logit), torch.empty_like(logit), None)
            gl, gq = coma_bwd_(logit, action, weight, adv, dq, T, B, A, N, upstream, spec)
        if need[6] and g_v is not None:
            g_ret = scale_(upstream[1], dret).view(T - 1, B * A)
        return (gl, gq, None, None, None, None, g_ret) + (None, ) * 6


# ----------------------------------------------------------------------------------------------------------------
# ScatterConnection (scatter_connection.py:59-121): csrc/scatter.cu.  x and the two index operands are read through their
# strides, so a permuted x or the location[..., 0] / [..., 1] views reach the kernels without a copy
# ----------------------------------------------------------------------------------------------------------------
SCATTER_MODES = {'add': 0, 'cover': 1}  # B200RL_SCATTER_ADD, B200RL_SCATTER_COVER


def scatter_fwd_(x, row, col, H, W, mode):
    """x (B, M, N) fp32, row / col (B, M) int64 (flat index col + row * W) -> the map (B, N, H, W)"""
    B, M, N = x.shape
    out = torch.empty(B, N, H, W, dtype=torch.float32, device=x.device)
    with on_device(x.device):
        rc = lib().b200rl_scatter_fwd(ptr(x), *x.stride(), ptr(row), *row.stride(), ptr(col), *col.stride(), B, M, N, H, W,
                                      mode, ptr(out), stream_ptr())
    _lib.check(rc, 'b200rl_scatter_fwd')
    return out


def scatter_bwd_(g, row, col, M, H, W):
    """g (B, N, H, W), the gradient of the map -> d x (B, M, N): g gathered at each entity's index (0 where it is out of
    range).  The kernels take the cell stride of g viewed as (B, N, H*W): reshape keeps g's memory when its H and W merge
    into one stride (an expanded gradient costs no copy) and copies otherwise.  The strides of size-1 dims do not describe
    the layout, so they are never read on their own: at W = 1 the cells step by g.stride(2)."""
    B, N = g.shape[0], g.shape[1]
    g = g.float().reshape(B, N, H * W)
    dx = torch.empty(B, M, N, dtype=torch.float32, device=g.device)
    with on_device(g.device):
        rc = lib().b200rl_scatter_bwd(ptr(g), *g.stride(), ptr(row), *row.stride(), ptr(col), *col.stride(), B, M, N, H, W,
                                      ptr(dx), stream_ptr())
    _lib.check(rc, 'b200rl_scatter_bwd')
    return dx


class ScatterFunction(torch.autograd.Function):
    """ScatterConnection's map from x; location gets no gradient.  One launch forward, one launch backward."""

    @staticmethod
    def forward(ctx, x, row, col, H, W, mode):
        ctx.save_for_backward(row, col)
        ctx.cfg = (x.shape[1], H, W)
        return scatter_fwd_(x, row, col, H, W, mode)

    @staticmethod
    def backward(ctx, g):
        row, col = ctx.saved_tensors
        dx = scatter_bwd_(g, row, col, *ctx.cfg) if ctx.needs_input_grad[0] else None
        return dx, None, None, None, None, None


# ----------------------------------------------------------------------------------------------------------------
# The layer-normalised LSTM (rnn.py:131-239, lstm_type='normal', norm_type='LN'): csrc/lstm.cu runs everything between
# the GEMMs, one launch per step in each direction; the GEMMs are torch.mm on the current stream (cuBLAS)
# ----------------------------------------------------------------------------------------------------------------
def _vec(t):
    return (ptr(t), t.stride(0))


def _mat(t):
    return (ptr(t), t.stride(0), t.stride(1))


_NO_MAT = (None, 0, 0)


def _rows_mm(a, b, T):
    """a @ b for the backward GEMMs whose rows are all T*B rows of a layer (dX, dWx, dWh).  At T = 1 they are the
    reference's own per-step shapes and run in fp32.  Above, they run in float64 and round once: on an H100 an fp32 cuBLAS
    GEMM of (1600, 512) x (512, 2048) measured about 5x the max error of a (64, 512) x (512, 2048) one, and in fp32 dX and
    dWx exceeded the reference's error after 25 and 80 steps."""
    if T == 1:
        return torch.mm(a, b)
    return torch.mm(a.double(), b.double()).float()


_F32 = 4  # bytes per element: the per-step operands are addressed as base pointer + offset, without a tensor view each


def lnlstm_fwd_(x, h0, c0, wx, wh, bias, gamma_x, beta_x, gamma_h, beta_h, save):
    """One layer over x (T, B, I) from the state h0, c0 (B, H) -> (y (T, B, H), h_T, c_T, GX, GH, C, stats).
    GX = x Wx (T, B, 4H) is one GEMM, in float64 rounded once at every T: in fp32, even at T = 1 where its shape is the
    reference's, 80 chained one-step calls (a recurrent learner's unroll) ended 3.6x further from float64 than the reference,
    with x Wx rounded once they stay within it.  GH[t] = h_{t-1} Wh is one fp32 GEMM per step.  C (T, B, H) holds
    c_1..c_T.  With ``save`` GH keeps every step and stats (T, B, 4) the LayerNorm statistics the backward reads; without
    it GH is one step's scratch and stats is None."""
    T, B, I = x.shape
    if T == 0:
        raise ValueError("di_engine_b200: the LSTM needs at least one time step (got an input of shape %s)" %
                         (tuple(x.shape), ))
    H = wh.shape[0]
    G = 4 * H
    GX = torch.mm(x.reshape(T * B, I).double(), wx.double()).float().view(T, B, G)
    y = GX.new_empty(T, B, H)
    hT = GX.new_empty(B, H)
    cT = GX.new_empty(B, H)
    C = GX.new_empty(T, B, H) if save or T > 1 else cT.view(1, B, H)  # c_1 of a one-step call without backward is c_T
    GH = GX.new_empty(T if save else 1, B, G)
    stats = GX.new_empty(T, B, 4) if save else None
    params = _vec(gamma_x) + _vec(beta_x) + _vec(gamma_h) + _vec(beta_h) + _vec(bias)
    p_gx, p_gh, p_y, p_c, p_st, p_ct = ptr(GX), ptr(GH), ptr(y), ptr(C), ptr(stats), ptr(cT)
    fn = lib().b200rl_lnlstm_step_fwd
    with on_device(x.device):
        st = stream_ptr()
        for t in range(T):
            last = t == T - 1
            s = t if save else 0
            torch.mm(h0 if t == 0 else y[t - 1], wh, out=GH[s])
            cp = _mat(c0) if t == 0 else (p_c + (t - 1) * B * H * _F32, H, 1)
            rc = fn(p_gx + t * B * G * _F32, G, 1, p_gh + s * B * G * _F32, G, 1, *params, *cp, B, H,
                    p_y + t * B * H * _F32, H, 1, p_c + t * B * H * _F32, H, 1, *(_mat(hT) if last else _NO_MAT),
                    *(_mat(cT) if last and C.data_ptr() != p_ct else _NO_MAT), p_st + t * B * 4 * _F32 if save else None,
                    4, st)
            _lib.check(rc, 'b200rl_lnlstm_step_fwd')
    return y, hT, cT, GX, GH, C, stats


def lnlstm_bwd_(g_y, g_hT, g_cT, x, h0, c0, wx, wh, bias, gamma_x, beta_x, gamma_h, beta_h, y, GX, GH, C, stats, needs):
    """The gradients of ``lnlstm_fwd_``'s (y, h_T, c_T) -> one per input (x, h0, c0, wx, wh, bias, gamma_x, beta_x, gamma_h,
    beta_h), None where ``needs`` is false.  Any upstream gradient may be None (zero).  One step launch per step, then
    dX = DGX Wx^T, dWx = X^T DGX, dWh = H_prev^T DGH over all T*B rows (``_rows_mm``) and one launch for the LayerNorm
    parameters."""
    T, B, I = x.shape
    H = wh.shape[0]
    G = 4 * H
    D = GX.new_empty(3, T, B, G)  # DGX, DGH, DG (the pre-activation's gradient)
    W = GX.new_empty(2, B, H)  # dc, and the recurrent term d_gh[t+1] Wh^T
    DGX, DGH = D[0], D[1]
    params = _vec(gamma_x) + _vec(beta_x) + _vec(gamma_h) + _vec(beta_h) + _vec(bias)
    p_d, p_w, p_gx, p_gh, p_c, p_st = ptr(D), ptr(W), ptr(GX), ptr(GH), ptr(C), ptr(stats)
    if g_y is not None:
        p_gy, gy_st = ptr(g_y), g_y.stride()
    L = lib()
    grads = [None] * 10
    with on_device(x.device):
        st = stream_ptr()
        for t in reversed(range(T)):
            if t == T - 1:
                rec = _mat(g_hT) if g_hT is not None else _NO_MAT
                dc_in = _mat(g_cT) if g_cT is not None else _NO_MAT
            else:
                torch.mm(DGH[t + 1], wh.t(), out=W[1])
                rec, dc_in = (p_w + B * H * _F32, H, 1), (p_w, H, 1)
            dy = (p_gy + t * gy_st[0] * _F32, gy_st[1], gy_st[2]) if g_y is not None else _NO_MAT
            cp = _mat(c0) if t == 0 else (p_c + (t - 1) * B * H * _F32, H, 1)
            step = t * B * G * _F32
            rc = L.b200rl_lnlstm_step_bwd(*dy, *rec, *dc_in, p_gx + step, G, 1, p_gh + step, G, 1,
                                          p_st + t * B * 4 * _F32, 4, *params, *cp, p_c + t * B * H * _F32, H, 1, B, H,
                                          p_d + step, G, 1, p_d + T * B * G * _F32 + step, G, 1,
                                          p_d + 2 * T * B * G * _F32 + step, G, 1, p_w, H, 1, st)
            _lib.check(rc, 'b200rl_lnlstm_step_bwd')
        dgx = DGX.view(T * B, G)
        if needs[0]:
            grads[0] = _rows_mm(dgx, wx.t(), T).view(T, B, I)
        if needs[1]:
            grads[1] = torch.mm(DGH[0], wh.t())
        if needs[2]:
            grads[2] = W[0]
        if needs[3]:
            grads[3] = _rows_mm(x.reshape(T * B, I).t(), dgx, T)
        if needs[4]:
            h_prev = h0 if T == 1 else torch.cat([h0.unsqueeze(0), y[:-1]]).view(T * B, H)
            grads[4] = _rows_mm(h_prev.t(), DGH.view(T * B, G), T)
        if any(needs[5:]):
            d_gamma_x, d_gamma_h, d_beta = (GX.new_empty(G) for _ in range(3))
            rc = L.b200rl_lnlstm_param_grads(p_d + 2 * T * B * G * _F32, G, 1, p_gx, G, 1, p_gh, G, 1, p_st, 4, T * B, H,
                                             *_vec(d_gamma_x), *_vec(d_gamma_h), *_vec(d_beta), st)
            _lib.check(rc, 'b200rl_lnlstm_param_grads')
            # bias, beta_x and beta_h all receive d_beta; each gets its own tensor, as autograd may keep one as a .grad
            grads[5:] = [d_beta, d_gamma_x, d_beta.clone(), d_gamma_h, d_beta.clone()]
    return [g if n else None for g, n in zip(grads, needs)]


class LNLSTMFunction(torch.autograd.Function):
    """One layer of the layer-normalised LSTM over a whole input sequence: (x (T, B, I), h0, c0 (B, H), wx, wh, bias[l],
    gamma_x, beta_x, gamma_h, beta_h, save) -> (y (T, B, H), h_T, c_T).  ``save`` (grad enabled and an input requires
    grad) keeps the backward's tensors; without it the forward keeps nothing beyond its own buffers."""

    @staticmethod
    def forward(ctx, x, h0, c0, wx, wh, bias, gamma_x, beta_x, gamma_h, beta_h, save):
        y, hT, cT, GX, GH, C, stats = lnlstm_fwd_(x, h0, c0, wx, wh, bias, gamma_x, beta_x, gamma_h, beta_h, save)
        if save:
            ctx.save_for_backward(x, h0, c0, wx, wh, bias, gamma_x, beta_x, gamma_h, beta_h, y, GX, GH, C, stats)
        ctx.set_materialize_grads(False)
        return y, hT, cT

    @staticmethod
    def backward(ctx, g_y, g_hT, g_cT):
        return tuple(lnlstm_bwd_(g_y, g_hT, g_cT, *ctx.saved_tensors, ctx.needs_input_grad[:10])) + (None, )


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
        ctx.factor = factor  # happo_error_continuous's per-sample factor (S,) or None; kept alive for the backward launch
        ctx.hint_kind = hint_kind
        ctx.cfg = (factor, S, D, clip_ratio, use_value_clip, dual_clip, kl_type)
        saved = (mu, sigma, value_new, mu_old, sigma_old, mu_pre, sigma_pre, action, value_old, adv, return_, weight)
        out, ctx.spec = ppoc_fwd_(saved, ctx.cfg, hint_kind, any(ctx.needs_input_grad[:3]))
        ctx.save_for_backward(*saved)
        ctx.set_materialize_grads(False)
        ctx.mark_non_differentiable(out)
        return out[0], out[1], out[2], out[3], out

    @staticmethod
    def backward(ctx, g_p, g_v, g_e, g_k, _g_out):
        keep, upstream = _grads(g_p, g_v, g_e, g_k)
        return ppoc_bwd_(ctx.saved_tensors, ctx.cfg, upstream, _forward_grads(ctx), ctx.hint_kind) + (None, ) * 17


def ppoc_fwd_(saved, cfg, hint_kind, want_grad):
    """The forward launch of ppo_error_continuous (PPOContinuousFunction and the ``b200rl::ppoc_loss`` custom op):
    ``saved`` = (mu, sigma, value_new, mu_old, sigma_old, mu_pre, sigma_pre, action, value_old, adv, return_, weight),
    ``cfg`` = (factor, S, D, clip_ratio, use_value_clip, dual_clip, kl_type).  -> (the 8-float result vector, the
    forward-written (grad_mu, grad_sigma, grad_value, g_used) or None without ``want_grad``)."""
    mu, sigma, value_new, mu_old, sigma_old, mu_pre, sigma_pre, action, value_old, adv, return_, weight = saved
    dev = mu.device
    out = torch.empty(8, dtype=torch.float32, device=dev)
    gm = torch.empty_like(mu) if want_grad else None
    gs = torch.empty_like(sigma) if want_grad else None
    gv = torch.empty_like(value_new) if want_grad else None
    g_used = torch.empty(4, dtype=torch.float32, device=dev) if want_grad else None
    hint = ppo_hint(dev, hint_kind)
    with on_device(dev):
        ws = workspace(dev)
        rc = lib().b200rl_ppo_continuous_fwd_grad(
            ptr(mu), ptr(sigma), ptr(mu_old), ptr(sigma_old), ptr(mu_pre), ptr(sigma_pre), ptr(action), ptr(value_new),
            ptr(value_old), ptr(adv), ptr(return_), ptr(weight), ptr(cfg[0]), *cfg[1:], ptr(hint) if want_grad else None,
            0, None, None, None, None, ptr(g_used), None, ptr(out), ptr(gm), ptr(gs), ptr(gv), ptr(ws), ws.numel() * 4,
            stream_ptr())
    _lib.check(rc, 'b200rl_ppo_continuous_fwd_grad')
    return out, (gm, gs, gv, g_used) if want_grad else None


def ppoc_bwd_(saved, cfg, upstream, spec, hint_kind):
    """The verify launch of ppo_error_continuous (arguments as ppoc_fwd_; ``upstream`` the four device pointers of the
    upstream gradients, None = 0).  With ``spec`` (the forward-written gradients) it verifies them on the device and
    recomputes them in place on a mismatch; without, it computes into fresh buffers.  -> (grad_mu, grad_sigma, grad_value)."""
    mu, sigma, value_new, mu_old, sigma_old, mu_pre, sigma_pre, action, value_old, adv, return_, weight = saved
    dev = mu.device
    gm, gs, gv, g_used = spec or (torch.empty_like(mu), torch.empty_like(sigma), torch.empty_like(value_new), None)
    with on_device(dev):
        ws = workspace(dev)
        rc = lib().b200rl_ppo_continuous_fwd_grad(
            ptr(mu), ptr(sigma), ptr(mu_old), ptr(sigma_old), ptr(mu_pre), ptr(sigma_pre), ptr(action), ptr(value_new),
            ptr(value_old), ptr(adv), ptr(return_), ptr(weight), ptr(cfg[0]), *cfg[1:], None, 1, *upstream, ptr(g_used),
            ptr(ppo_hint(dev, hint_kind)), None, ptr(gm), ptr(gs), ptr(gv), ptr(ws), ws.numel() * 4, stream_ptr())
    _lib.check(rc, 'b200rl_ppo_continuous_fwd_grad(verify)')
    return gm, gs, gv


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
        scal = (gamma, lambda_, rho_clip, c_clip, rho_pg_clip)
        out, fused, spec, cpg, dv = vtrace_fwd_(target_output, value, behaviour_output, action, reward, weight, scal,
                                                ctx.needs_input_grad[0] or ctx.needs_input_grad[1])
        ctx.scal = scal if fused else None  # the scalars of the verify launch: set on the one-launch path only
        if fused:
            ctx.spec = spec
            ctx.save_for_backward(target_output, behaviour_output, action, value, reward, weight)
        else:
            ctx.save_for_backward(target_output, action, weight, cpg, dv)
        return out[0], out[1], out[2]

    @staticmethod
    def backward(ctx, g_p, g_v, g_e):
        keep, upstream = _grads(g_p, g_v, g_e)
        if ctx.scal is not None:
            grads = vtrace_verify_(ctx.saved_tensors, ctx.scal, upstream, _forward_grads(ctx))
        else:
            target_output, action, weight, cpg, dv = ctx.saved_tensors
            grads = vtrace_bwd_(target_output, action, weight, cpg, dv, upstream)
        return grads + (None, ) * 9


def vtrace_fwd_(target_output, value, behaviour_output, action, reward, weight, scal, want_grad):
    """The forward launch of vtrace_error_discrete_action (VTraceFunction and the ``b200rl::vtrace_loss`` custom op); ``scal``
    = (gamma, lambda_, rho_clip, c_clip, rho_pg_clip).  -> (out, fused, spec, cpg, dv): ``fused`` when the one-launch kernel
    ran, with ``spec`` its forward-written (grad_logit, grad_value, g_used) when ``want_grad``; otherwise the rows / scan
    kernels ran and ``cpg`` / ``dv`` are the (T, B) records of their backward."""
    T, B = reward.shape
    N = target_output.shape[-1]
    dev = target_output.device
    out = torch.empty(4, dtype=torch.float32, device=dev)
    L = lib()
    tensors = (ptr(target_output), ptr(behaviour_output), ptr(action), ptr(value), ptr(reward), ptr(weight))
    with on_device(dev):
        ws = workspace(dev)
        if VTRACE_FUSED:
            grad_logit = torch.empty_like(target_output) if want_grad else None
            grad_value = torch.empty(T + 1, B, dtype=torch.float32, device=dev) if want_grad else None
            if L.b200rl_vtrace_fused_supported(*tensors, T, B, N, ptr(grad_logit), ptr(grad_value)):
                g_used = torch.empty(3, dtype=torch.float32, device=dev) if want_grad else None
                rc = L.b200rl_vtrace_fwd_grad(
                    *tensors, T, B, N, *scal, ptr(vtrace_hint(dev)) if want_grad else None, 0, None, None, None,
                    ptr(g_used), None, ptr(out), ptr(grad_logit), ptr(grad_value), ptr(ws), ws.numel() * 4, stream_ptr()
                )
                _lib.check(rc, 'b200rl_vtrace_fwd_grad')
                return out, True, (grad_logit, grad_value, g_used) if want_grad else None, None, None
        lp = torch.empty(T, B, dtype=torch.float32, device=dev)
        cpg = torch.empty(T, B, dtype=torch.float32, device=dev)
        dv = torch.empty(T, B, dtype=torch.float32, device=dev)
        rc = L.b200rl_vtrace_fwd(
            *tensors, T, B, N, *scal, ptr(out), ptr(lp), ptr(cpg), ptr(dv), ptr(ws), ws.numel() * 4, stream_ptr()
        )
    _lib.check(rc, 'b200rl_vtrace_fwd')
    return out, False, None, cpg, dv


def vtrace_verify_(saved, scal, upstream, spec):
    """The backward launch after a one-launch forward: ``saved`` = (target_output, behaviour_output, action, value, reward,
    weight), ``upstream`` the three device pointers of the upstream gradients (None = 0).  With ``spec`` it verifies the
    forward-written gradients on the device (recomputing in place on a mismatch), else it recomputes into fresh buffers.
    -> (grad_logit, grad_value)."""
    target_output, behaviour_output, action, value, reward, weight = saved
    T, B = reward.shape
    N = target_output.shape[-1]
    dev = target_output.device
    grad_logit, grad_value, g_used = spec or (
        torch.empty_like(target_output), torch.empty(T + 1, B, dtype=torch.float32, device=dev), None)
    with on_device(dev):
        ws = workspace(dev)
        rc = lib().b200rl_vtrace_fwd_grad(
            ptr(target_output), ptr(behaviour_output), ptr(action), ptr(value), ptr(reward), ptr(weight), T, B,
            N, *scal, None, 1, *upstream, ptr(g_used), ptr(vtrace_hint(dev)), None, ptr(grad_logit),
            ptr(grad_value), ptr(ws), ws.numel() * 4, stream_ptr()
        )
    _lib.check(rc, 'b200rl_vtrace_fwd_grad(verify)')
    return grad_logit, grad_value


def vtrace_bwd_(target_output, action, weight, cpg, dv, upstream):
    """The backward launch after the rows / scan forward -> (grad_logit, grad_value)."""
    T, B = cpg.shape
    N = target_output.shape[-1]
    dev = target_output.device
    grad_logit = torch.empty_like(target_output)
    grad_value = torch.empty(T + 1, B, dtype=torch.float32, device=dev)
    with on_device(dev):
        rc = lib().b200rl_vtrace_bwd(
            ptr(target_output), ptr(action), ptr(weight), ptr(cpg), ptr(dv), *upstream, T, B, N, ptr(grad_logit),
            ptr(grad_value), stream_ptr()
        )
    _lib.check(rc, 'b200rl_vtrace_bwd')
    return grad_logit, grad_value


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


def _vocab_rows(dev, rows):
    """the per-call outputs of a GRPO / RLOO launch: the three loss sums, logsumexp and the unit coefficient per row"""
    return (torch.empty(3, dtype=torch.float32, device=dev), torch.empty(rows, dtype=torch.float32, device=dev),
            torch.empty(rows, dtype=torch.float32, device=dev))


def grpo_fwd_(logit_new, logit_old, logit_ref, action, adv, weight, dt, clip_ratio, beta, grad):
    """The forward launch of grpo_policy_error (GRPOFunction and the ``b200rl::lm_policy_fwd`` custom op): logits
    (B, S, V) contiguous and 16-byte aligned.  -> (loss / approx_kl / clipfrac, logsumexp of logit_new per row, d loss /
    d lp_new per row for a unit upstream gradient); also writes d loss / d logit_new for that gradient into ``grad``
    unless it is None."""
    B, S, V = logit_new.shape
    dev = logit_new.device
    out, lse, dlp = _vocab_rows(dev, B * S)
    with on_device(dev):
        ws = workspace(dev)
        rc = lib().b200rl_grpo_fwd_grad(dt, ptr(logit_new), ptr(logit_old), ptr(logit_ref), ptr(action), ptr(adv),
                                        ptr(weight), B, S, V, clip_ratio, beta, ptr(out), ptr(lse), ptr(dlp),
                                        ptr(grad), ptr(ws), ws.numel() * 4, stream_ptr())
    _lib.check(rc, 'b200rl_grpo_fwd_grad')
    return out, lse, dlp


def rloo_fwd_(logit_new, logit_old, action, reward, weight, dt, clip_ratio, grad):
    """The forward launch of rloo_policy_error, reward (K, B / K); as ``grpo_fwd_``"""
    B, S, V = logit_new.shape
    dev = logit_new.device
    out, lse, dlp = _vocab_rows(dev, B * S)
    with on_device(dev):
        ws = workspace(dev)
        rc = lib().b200rl_rloo_fwd_grad(dt, ptr(logit_new), ptr(logit_old), ptr(action), ptr(reward), reward.shape[0],
                                        ptr(weight), B, S, V, clip_ratio, ptr(out), ptr(lse), ptr(dlp), ptr(grad),
                                        ptr(ws), ws.numel() * 4, stream_ptr())
    _lib.check(rc, 'b200rl_rloo_fwd_grad')
    return out, lse, dlp


class GRPOFunction(torch.autograd.Function):
    """grpo_policy_error (ding/rl_utils/grpo.py) on logits (B, S, V): outputs loss (differentiable w.r.t. logit_new),
    approx_kl and clipfrac.  ONE forward launch (+ the loss-sum finalize) also writes d loss / d logit_new for a unit
    upstream gradient; ``backward`` hands that buffer to autograd after a launch that returns at once on the device when
    the upstream gradient really is 1, and recomputes otherwise from the saved per-row logsumexp and coefficient."""

    @staticmethod
    def forward(ctx, logit_new, logit_old, logit_ref, action, adv, weight, dt, clip_ratio, beta):
        grad = torch.empty_like(logit_new) if ctx.needs_input_grad[0] else None
        out, lse, dlp = grpo_fwd_(logit_new, logit_old, logit_ref, action, adv, weight, dt, clip_ratio, beta, grad)
        return _vocab_saved(ctx, logit_new, action, lse, dlp, grad, dt, out)

    @staticmethod
    def backward(ctx, g_loss, _g_kl, _g_cf):
        return (_vocab_backward(ctx, g_loss), ) + (None, ) * 8


class RLOOFunction(torch.autograd.Function):
    """rloo_policy_error (ding/rl_utils/rloo.py) on logits (B, S, V); the leave-one-out advantage is formed in the kernel
    from reward (K, B / K).  Outputs and backward as ``GRPOFunction``."""

    @staticmethod
    def forward(ctx, logit_new, logit_old, action, reward, weight, dt, clip_ratio):
        grad = torch.empty_like(logit_new) if ctx.needs_input_grad[0] else None
        out, lse, dlp = rloo_fwd_(logit_new, logit_old, action, reward, weight, dt, clip_ratio, grad)
        return _vocab_saved(ctx, logit_new, action, lse, dlp, grad, dt, out)

    @staticmethod
    def backward(ctx, g_loss, _g_kl, _g_cf):
        return (_vocab_backward(ctx, g_loss), ) + (None, ) * 6


def ppo_lm_fwd_(logit_new, logit_old, logit_pre, action, adv, weight, dt, clip_ratio, dual_clip, kl_type, entropy, hint,
                grad, g_used):
    """The forward launch of ppo_policy_error on token rows (PPOLMFunction and the ``b200rl::ppo_lm_fwd`` custom op).
    -> (the five loss sums, and per row: logsumexp, entropy (None without ``entropy``), the policy term's unit coefficient,
    the kl term's (None without logit_pre)).  With ``grad`` it also writes d / d logit_new for the upstream gradients of
    the record ``hint`` and records them in ``g_used``."""
    dev = logit_new.device
    V = logit_new.shape[-1]
    rows = logit_new.numel() // V
    out = torch.empty(5, dtype=torch.float32, device=dev)
    lse = torch.empty(rows, dtype=torch.float32, device=dev)
    ent = torch.empty(rows, dtype=torch.float32, device=dev) if entropy else None
    dpol = torch.empty(rows, dtype=torch.float32, device=dev)
    dkl = torch.empty(rows, dtype=torch.float32, device=dev) if logit_pre is not None else None
    with on_device(dev):
        ws = workspace(dev)
        rc = lib().b200rl_ppo_lm_fwd_grad(
            dt, ptr(logit_new), ptr(logit_old), ptr(logit_pre), ptr(action), ptr(adv), ptr(weight), rows, V,
            clip_ratio, dual_clip, kl_type, 1 if entropy else 0, ptr(hint), ptr(g_used), ptr(out), ptr(lse), ptr(ent),
            ptr(dpol), ptr(dkl), ptr(grad), ptr(ws), ws.numel() * 4, stream_ptr())
    _lib.check(rc, 'b200rl_ppo_lm_fwd_grad')
    return out, lse, ent, dpol, dkl


def ppo_lm_bwd_(dt, logit_new, action, weight, lse, ent, dpol, dkl, upstream, g_used, hint, grad):
    """The backward launch of ppo_policy_error on token rows: ``upstream`` the device pointers of the policy, entropy and
    kl upstream gradients (None = 0).  With ``g_used`` (the forward-written gradient's record) it returns at once on the
    device when they match it and rewrites ``grad`` otherwise; without, it computes ``grad``.  -> grad."""
    with on_device(logit_new.device):
        rc = lib().b200rl_ppo_lm_bwd(dt, ptr(logit_new), ptr(action), ptr(weight), lse.numel(), logit_new.shape[-1],
                                     ptr(lse), ptr(ent), ptr(dpol), ptr(dkl), *upstream, ptr(g_used), ptr(hint),
                                     ptr(grad), stream_ptr())
    _lib.check(rc, 'b200rl_ppo_lm_bwd')
    return grad


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
        want = ctx.needs_input_grad[0]
        grad = torch.empty_like(logit_new) if want else None
        g_used = torch.empty(4, dtype=torch.float32, device=dev) if want else None
        ctx.hint_kind = hint_kind
        out, lse, ent, dpol, dkl = ppo_lm_fwd_(logit_new, logit_old, logit_pre, action, adv, weight, dt, clip_ratio,
                                               dual_clip, kl_type, entropy, ppo_hint(dev, hint_kind) if want else None,
                                               grad, g_used)
        ctx.save_for_backward(logit_new, action, weight, lse, ent, dpol, dkl)
        ctx.dt = dt
        ctx.spec = (grad, g_used) if want else None
        ctx.mark_non_differentiable(out)
        return out[0], out[1], out[2], out

    @staticmethod
    def backward(ctx, g_p, g_e, g_k, _g_out):
        logit_new, action, weight, lse, ent, dpol, dkl = ctx.saved_tensors
        keep, upstream = _grads(g_p, g_e, g_k)
        spec = _forward_grads(ctx)
        if spec is not None:  # valid if the expectation held; the kernel checks on the device
            grad, g_used = spec
            hint = ppo_hint(logit_new.device, ctx.hint_kind)
        else:  # a repeated backward: null g_used / hint -> the kernel recomputes
            grad, g_used, hint = torch.empty_like(logit_new), None, None
        grad = ppo_lm_bwd_(ctx.dt, logit_new, action, weight, lse, ent, dpol, dkl, upstream, g_used, hint, grad)
        return (grad, ) + (None, ) * 11


def a2c_lm_fwd_(logit, value, action, adv, return_, weight, dt, hint, gl, gv, g_used):
    """The forward launch of a2c_error on token rows (A2CLMFunction and the ``b200rl::a2c_lm_fwd`` custom op).  -> (the
    three loss sums, (4, rows): per row logsumexp, entropy, the policy term's unit coefficient, d value_loss / d value).  With
    ``gl`` / ``gv`` it also writes d / d logit and d / d value for the upstream gradients of the record ``hint`` and records
    them in ``g_used``."""
    dev = logit.device
    V = logit.shape[-1]
    rows = logit.numel() // V
    out = torch.empty(3, dtype=torch.float32, device=dev)
    per_row = torch.empty(4, rows, dtype=torch.float32, device=dev)
    lse, ent, dpol, dval = per_row.unbind(0)
    with on_device(dev):
        ws = workspace(dev)
        rc = lib().b200rl_a2c_lm_fwd_grad(
            dt, ptr(logit), ptr(action), ptr(value), ptr(adv), ptr(return_), ptr(weight), rows, V, ptr(hint),
            ptr(g_used), ptr(out), ptr(lse), ptr(ent), ptr(dpol), ptr(dval), ptr(gl), ptr(gv), ptr(ws), ws.numel() * 4,
            stream_ptr())
    _lib.check(rc, 'b200rl_a2c_lm_fwd_grad')
    return out, per_row


def a2c_lm_bwd_(dt, logit, action, weight, lse, ent, dpol, dval, upstream, g_used, hint, gl, gv):
    """The backward launch of a2c_error on token rows: ``upstream`` the device pointers of the policy, value and entropy
    upstream gradients (None = 0); with ``g_used`` it verifies as ``ppo_lm_bwd_``.  -> (gl, gv)."""
    with on_device(logit.device):
        rc = lib().b200rl_a2c_lm_bwd(dt, ptr(logit), ptr(action), ptr(weight), lse.numel(), logit.shape[-1], ptr(lse),
                                     ptr(ent), ptr(dpol), ptr(dval), *upstream, ptr(g_used), ptr(hint), ptr(gl),
                                     ptr(gv), stream_ptr())
    _lib.check(rc, 'b200rl_a2c_lm_bwd')
    return gl, gv


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
        want = ctx.needs_input_grad[0] or ctx.needs_input_grad[1]
        gl = torch.empty_like(logit) if want else None
        gv = torch.empty_like(value) if want else None
        g_used = torch.empty(4, dtype=torch.float32, device=dev) if want else None
        out, per_row = a2c_lm_fwd_(logit, value, action, adv, return_, weight, dt, ppo_hint(dev, 'a2c') if want else None,
                                   gl, gv, g_used)
        ctx.save_for_backward(logit, value, action, weight, *per_row.unbind(0))
        ctx.dt = dt
        ctx.spec = (gl, gv, g_used) if want else None
        ctx.set_materialize_grads(False)
        return out[0], out[1], out[2]

    @staticmethod
    def backward(ctx, g_p, g_v, g_e):
        logit, value, action, weight, lse, ent, dpol, dval = ctx.saved_tensors
        keep, upstream = _grads(g_p, g_v, g_e)
        spec = _forward_grads(ctx)
        if spec is not None:  # valid if the expectation held; the kernel checks on the device
            gl, gv, g_used = spec
            hint = ppo_hint(logit.device, 'a2c')
        else:  # a repeated backward: null g_used / hint -> the kernel recomputes
            gl, gv, g_used, hint = torch.empty_like(logit), torch.empty_like(value), None, None
        gl, gv = a2c_lm_bwd_(ctx.dt, logit, action, weight, lse, ent, dpol, dval, upstream, g_used, hint, gl, gv)
        return gl, gv, None, None, None, None, None


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
    return token_logp_bwd_(ctx.dt, logit_new, action, lse, dlp, pg, skip, grad)


def token_logp_fwd_(dt, logits, index):
    """The forward launch of the log-prob methods: logits (rows, V) -> (log p(index), logsumexp) per row, fp32"""
    rows = logits.shape[0]
    lp = torch.empty(rows, dtype=torch.float32, device=logits.device)
    lse = torch.empty(rows, dtype=torch.float32, device=logits.device)
    with on_device(logits.device):
        rc = lib().b200rl_token_logp_fwd(dt, ptr(logits), ptr(index), rows, logits.shape[-1], ptr(lp), ptr(lse),
                                         stream_ptr())
    _lib.check(rc, 'b200rl_token_logp_fwd')
    return lp, lse


def token_logp_bwd_(dt, logits, index, lse, coef, pg, skip, grad):
    """The backward launch of the vocabulary rows: ``grad`` = (*pg, or 1 for a null pg) * coef[row] * (onehot(index) -
    softmax(logits[row])), the gradient of the log-prob methods (coef = their upstream gradient) and of GRPO / RLOO (coef
    = the unit coefficient).  With ``skip`` the launch returns at once on the device when *pg is 1: ``grad`` then holds
    the forward-written gradient.  -> grad."""
    with on_device(logits.device):
        rc = lib().b200rl_token_logp_bwd(dt, ptr(logits), ptr(index), ptr(lse), ptr(coef), pg, skip, lse.numel(),
                                         logits.shape[-1], ptr(grad), stream_ptr())
    _lib.check(rc, 'b200rl_token_logp_bwd')
    return grad


class TokenLogProbFunction(torch.autograd.Function):
    """log p(index) under softmax(logits) per token (ding/rl_utils/log_prob_utils.py): logits (rows, V) fp32 or bf16,
    index (rows) -> fp32 (rows).  Backward: d / d logits = g * (onehot - softmax), one launch."""

    @staticmethod
    def forward(ctx, logits, index, dt):
        lp, lse = token_logp_fwd_(dt, logits, index)
        ctx.save_for_backward(logits, index, lse)
        ctx.dt = dt
        return lp

    @staticmethod
    def backward(ctx, g):
        logits, index, lse = ctx.saved_tensors
        g = g.float().contiguous()
        return token_logp_bwd_(ctx.dt, logits, index, lse, g, None, 0, torch.empty_like(logits)), None, None


def token_head_fwd_(lp_new, lp_old, lp_ref, adv, reward, weight, clip_ratio, beta):
    """The one launch of the GRPO (``lp_ref`` given) or RLOO head on per-token log-probabilities (B, S) fp32: -> (loss /
    approx_kl / clipfrac, d loss / d lp_new (B, S) for a unit upstream gradient)"""
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
    return out, dlp


def token_head_(lp_new, lp_old, lp_ref, adv, reward, weight, clip_ratio, beta):
    """The GRPO (``lp_ref`` given) or RLOO head on per-token log-probabilities (B, S) fp32 from a caller's own
    log_prob_fn: returns (loss, approx_kl, clipfrac); the gradient reaches ``lp_new`` (b200rl_scale of the saved
    unit-upstream gradient), and through it whatever computed it."""
    out, dlp = token_head_fwd_(lp_new, lp_old, lp_ref, adv, reward, weight, clip_ratio, beta)
    loss = out[0]
    if lp_new.requires_grad and torch.is_grad_enabled():
        loss = _ScaleSaved.apply(lp_new, loss, dlp)
    return loss, out[1], out[2]


# ----------------------------------------------------------------------------------------------------------------
# GRPO / RLOO / per-token log p from the lm_head's hidden states (rl_utils/lm_linear.py): the logits exist one chunk of
# token rows at a time (cuBLAS through torch.mm, with the caller's matmul precision settings, as F.linear), and the row
# work runs in place on the chunk (csrc/vocab.cu, b200rl_lm_linear_fwd / _bwd)
# ----------------------------------------------------------------------------------------------------------------
# Bytes of the one (rows_per_chunk, V) logit buffer of a call.  Chosen by measurement (tools/bench_lm_linear.py --budgets,
# one H100 80GB HBM3 at 700 W, 16 x 1024 tokens, D = 3584, V = 152 064 bf16): GRPO forward + backward took 147 / 114 /
# 98 / 90 ms at 128 / 256 / 512 / 1024 MiB, because the dW GEMM's inner dimension is the chunk's rows and short chunks
# leave it far from peak (390 -> 700 TFLOP/s over the three GEMMs).  Up to 1 GiB the call's peak memory did not move
# (3.39 GB: the fp32 dW accumulator and the rounded dW, which coexist after the last chunk, outweigh the chunk).
# Module-level so that a test can shrink it to force many chunks.
LM_CHUNK_BYTES = 1 << 30
_LM_MODE = {'grpo': 0, 'rloo': 1, 'logp': 2, 'ppo': 3, 'a2c': 4}  # B200RL_LM_GRPO .. B200RL_LM_A2C
_VOCAB_CTAS_PER_SM = 4  # vocab_rows_kernel: 512 threads, at most 2048 resident per SM
_WS_PARTIAL_WORDS = 256000 - 16  # WS_PARTIAL_LIMIT_WORDS - WS_CTRL_WORDS (csrc/common.cuh)


def sm_count(device):
    return torch.cuda.get_device_properties(device).multi_processor_count


def lm_chunk_plan(N, V, itemsize, sms, loss, sums=3):
    """(rows per chunk, chunks) for N token rows of V logits of ``itemsize`` bytes: the largest multiple of 128 rows whose
    logits fit in LM_CHUNK_BYTES (at least 128), or all N rows when there are fewer.  A loss call stores ``sums`` partial
    sums (GRPO / RLOO / A2C 3, PPO 5) per CTA per chunk (at most sms * 4 CTAs, and no more than the chunk's rows); raises
    before any launch when they would not fit in the workspace."""
    rows = min(N, max(128, LM_CHUNK_BYTES // (V * itemsize) // 128 * 128))
    n = -(-N // rows)
    if loss and n * min(rows, sms * _VOCAB_CTAS_PER_SM) * sums > _WS_PARTIAL_WORDS:
        raise ValueError("di_engine_b200: %d token rows in %d chunks of %d need more loss partials than the workspace "
                         "holds; raise ops.LM_CHUNK_BYTES" % (N, n, rows))
    return rows, n


def _acc_dw(acc, z, h):
    """acc (V, D) fp32 += z^T h: fp32 accumulation of the chunks' dW whatever the GEMM operands' dtype"""
    if z.dtype == torch.float32:
        acc.addmm_(z.t(), h)
    else:
        torch.addmm(acc, z.t(), h, out_dtype=torch.float32, out=acc)


def _dw_out(acc, dtype):
    """the fp32 dW accumulator rounded once to the weight's dtype"""
    return acc if acc is None or acc.dtype == dtype else acc.to(dtype)


def lm_chunks_(hidden, lm_weight, rows, n, launch, want_dh, want_dw):
    """The chunk loop of every hidden-state loss: hidden (N, D) and lm_weight (V, D), both contiguous and of one dtype,
    in ``n`` chunks of ``rows`` token rows through one (rows, V) buffer z.  Per chunk: the logit GEMM z = H[chunk] W^T,
    ``launch(z, r0)`` (the row launch, which overwrites z in place with d loss / d logits when a gradient is wanted), then
    dH[chunk] = z W only if ``want_dh`` and dW += z^T H[chunk] (fp32) only if ``want_dw``.  -> (dH or None, dW rounded
    once to the weight's dtype, or None)."""
    N, D = hidden.shape
    V = lm_weight.shape[0]
    dev = hidden.device
    z = torch.empty(rows, V, dtype=hidden.dtype, device=dev)
    dh = torch.empty_like(hidden) if want_dh else None
    acc = torch.zeros(V, D, dtype=torch.float32, device=dev) if want_dw else None
    wt = lm_weight.t()
    for c in range(n):
        r0 = c * rows
        zc, hc = z[:min(rows, N - r0)], hidden[r0:r0 + rows]
        torch.mm(hc, wt, out=zc)
        launch(zc, r0)
        if want_dh:
            torch.mm(zc, lm_weight, out=dh[r0:r0 + rows])
        if want_dw:
            _acc_dw(acc, zc, hc)
    del z, zc
    return dh, _dw_out(acc, hidden.dtype)


def lm_linear_loss_(hidden, lm_weight, action, lp_old, lp_ref, side, weight, kind, B, S, dt, clip_ratio, beta, want_dh,
                    want_dw):
    """GRPO (``kind`` 'grpo', side = adv (B)) or RLOO ('rloo', side = reward (K, B / K)) on hidden (N = B*S, D) and
    lm_weight (V, D), both contiguous and of one dtype; action, lp_old, lp_ref (N), weight (N) or None.  ``lm_chunks_``
    with the GRPO / RLOO row launch.  -> (out3 = loss / approx_kl / clipfrac, dH or None, dW or None)."""
    N = hidden.shape[0]
    V = lm_weight.shape[0]
    dev = hidden.device
    rows, n = lm_chunk_plan(N, V, hidden.element_size(), sm_count(dev), True)
    want = want_dh or want_dw
    grpo = kind == 'grpo'
    out = torch.empty(3, dtype=torch.float32, device=dev)
    lse = torch.empty(N, dtype=torch.float32, device=dev)
    seq = torch.empty(2 * B, dtype=torch.float32, device=dev)
    with on_device(dev):
        ws = workspace(dev)
        L, st = lib(), stream_ptr()

        def launch(zc, r0):
            rc = L.b200rl_lm_linear_fwd(_LM_MODE[kind], dt, ptr(zc), r0, zc.shape[0], rows, V, B, S, ptr(action),
                                        ptr(lp_old), ptr(lp_ref), ptr(side) if grpo else None,
                                        None if grpo else ptr(side), 0 if grpo else side.shape[0], ptr(weight), ptr(seq),
                                        clip_ratio, beta, None, ptr(lse), ptr(out), 1 if want else 0, ptr(ws),
                                        ws.numel() * 4, st)
            _lib.check(rc, 'b200rl_lm_linear_fwd')

        dh, dw = lm_chunks_(hidden, lm_weight, rows, n, launch, want_dh, want_dw)
    return out, dh, dw


def lm_linear_pg_(hidden, lm_weight, action, adv, weight, lp_old, lp_pre, value, ret, kind, dt, cfg, want_dh, want_dw,
                  want_dv):
    """PPO (``kind`` 'ppo': lp_old (N), lp_pre (N) or None) or A2C ('a2c': value, ret (N)) on hidden (N = B*S, D) and
    lm_weight (V, D), both contiguous and of one dtype; action, adv (N), weight (N) or None.  cfg = (clip_ratio,
    dual_clip (0 = off), kl_type, entropy, w_ent, w_kl, w_val): the loss is policy + w_val * value + w_ent * entropy +
    w_kl * kl.  ``lm_chunks_`` with the PPO / A2C row launch, whose forward-written gradients are for a unit upstream
    gradient of that loss.  -> (out: PPO's five sums policy / entropy / kl / approx_kl / clipfrac, A2C's three policy /
    value / entropy; dH or None; dW or None; d value (N) fp32 or None)."""
    N = hidden.shape[0]
    V = lm_weight.shape[0]
    dev = hidden.device
    ppo = kind == 'ppo'
    rows, n = lm_chunk_plan(N, V, hidden.element_size(), sm_count(dev), True, 5 if ppo else 3)
    want = want_dh or want_dw
    clip_ratio, dual_clip, kl_type, entropy, w_ent, w_kl, w_val = cfg
    out = torch.empty(5 if ppo else 3, dtype=torch.float32, device=dev)
    dv = torch.empty(N, dtype=torch.float32, device=dev) if want_dv else None
    with on_device(dev):
        ws = workspace(dev)
        L, st = lib(), stream_ptr()

        def launch(zc, r0):
            rc = L.b200rl_lm_linear_pg_fwd(_LM_MODE[kind], dt, ptr(zc), r0, zc.shape[0], rows, V, N, ptr(action),
                                           ptr(lp_old), ptr(lp_pre), ptr(adv), ptr(value), ptr(ret), ptr(weight),
                                           clip_ratio, dual_clip, kl_type, 1 if entropy else 0, w_ent, w_kl, w_val,
                                           ptr(dv), ptr(out), 1 if want else 0, ptr(ws), ws.numel() * 4, st)
            _lib.check(rc, 'b200rl_lm_linear_pg_fwd')

        dh, dw = lm_chunks_(hidden, lm_weight, rows, n, launch, want_dh, want_dw)
    return out, dh, dw, dv


def lm_scale_(dt, pg, x):
    """x *= *pg in place, skipped on the device when *pg == 1 (the forward wrote x for a unit upstream gradient)"""
    with on_device(x.device):
        rc = lib().b200rl_lm_linear_scale(dt, pg, ptr(x), x.numel(), stream_ptr())
    _lib.check(rc, 'b200rl_lm_linear_scale')
    return x


def lm_scale_out_(dt, pg, x):
    """*pg * x into a fresh tensor, the bits of ``lm_scale_`` (x's own when *pg == 1): the backward op of the hidden-state
    losses under torch.compile, which may not hand back the buffer its forward op wrote.  The kernel reads x.numel()
    values from x's address, so a strided view is made contiguous first."""
    x = x.contiguous()
    out = torch.empty_like(x)
    with on_device(x.device):
        rc = lib().b200rl_lm_linear_scale_out(dt, pg, ptr(x), ptr(out), x.numel(), stream_ptr())
    _lib.check(rc, 'b200rl_lm_linear_scale_out')
    return out


def _lm_backward(ctx, g_loss, recompute):
    """The backward of the hidden-state losses: the gradients their forward wrote for a unit upstream gradient of the one
    loss (``ctx.spec``; dH, dW and, for A2C, d value), scaled in place by ``g_loss`` on the device (a no-op when it is 1).
    A repeated backward gets them from ``recompute()`` instead, since the first one handed the forward's buffers out."""
    spec = _forward_grads(ctx)
    grads = recompute() if spec is None else spec
    keep, (pg, ) = _grads(g_loss)
    for x in grads:
        if x is not None:
            lm_scale_(_LOGIT_DTYPES[x.dtype], pg, x)
    return grads


class LMLinearLossFunction(torch.autograd.Function):
    """grpo_policy_error_linear / rloo_policy_error_linear: outputs loss (differentiable w.r.t. hidden and lm_weight),
    approx_kl and clipfrac.  The forward also writes dH and dW for a unit upstream gradient, each only if its input
    requires grad; ``backward`` hands them to autograd, scaled in place by the upstream gradient on the device (a no-op
    when it is 1).  A repeated backward recomputes them."""

    @staticmethod
    def forward(ctx, hidden, lm_weight, action, lp_old, lp_ref, side, weight, kind, B, S, dt, clip_ratio, beta):
        want = ctx.needs_input_grad[:2]
        out, dh, dw = lm_linear_loss_(hidden, lm_weight, action, lp_old, lp_ref, side, weight, kind, B, S, dt,
                                      clip_ratio, beta, *want)
        ctx.save_for_backward(hidden, lm_weight, action, lp_old, lp_ref, side, weight)
        ctx.cfg = (kind, B, S, dt, clip_ratio, beta)
        ctx.spec = (dh, dw)
        ctx.set_materialize_grads(False)
        loss, approx_kl, clipfrac = out[0], out[1], out[2]
        ctx.mark_non_differentiable(approx_kl, clipfrac)
        return loss, approx_kl, clipfrac

    @staticmethod
    def backward(ctx, g_loss, _g_kl, _g_cf):
        if g_loss is None:
            return (None, ) * 13

        def recompute():
            hidden, lm_weight, *rest = ctx.saved_tensors
            return lm_linear_loss_(hidden, lm_weight, *rest, *ctx.cfg, *ctx.needs_input_grad[:2])[1:]

        return tuple(_lm_backward(ctx, g_loss, recompute)) + (None, ) * 11


def lm_pg_loss_(out, kind, cfg):
    """the one loss of ``lm_linear_pg_``'s sums: PPO policy + w_ent * entropy + w_kl * kl, A2C policy + w_val * value +
    w_ent * entropy (fp32, left to right; a zero weight adds nothing)"""
    _, _, _, _, w_ent, w_kl, w_val = cfg
    loss = out[0].clone()
    for k, wk in enumerate((w_ent, w_kl) if kind == 'ppo' else (w_val, w_ent), 1):
        if wk != 0.0:
            loss = loss + wk * out[k]
    return loss


class LMLinearPGFunction(torch.autograd.Function):
    """ppo_policy_error_linear / a2c_error_linear: outputs the one loss (policy + w_val * value + w_ent * entropy + w_kl *
    kl; differentiable w.r.t. hidden, lm_weight and, for A2C, value) and the raw result vector (non differentiable: PPO's
    policy / entropy / kl / approx_kl / clipfrac, A2C's policy / value / entropy).  The forward also writes dH, dW and
    d value for a unit upstream gradient of the loss, each only if its input requires grad; ``backward`` is
    ``LMLinearLossFunction``'s: scaled in place, recomputed on a repeated backward."""

    @staticmethod
    def forward(ctx, hidden, lm_weight, value, action, adv, weight, lp_old, lp_pre, ret, kind, dt, cfg):
        want = ctx.needs_input_grad[:3]
        out, dh, dw, dv = lm_linear_pg_(hidden, lm_weight, action, adv, weight, lp_old, lp_pre, value, ret, kind, dt,
                                        cfg, *want)
        ctx.save_for_backward(hidden, lm_weight, value, action, adv, weight, lp_old, lp_pre, ret)
        ctx.cfg = (kind, dt, cfg)
        ctx.spec = (dh, dw, dv)
        ctx.set_materialize_grads(False)
        ctx.mark_non_differentiable(out)
        return lm_pg_loss_(out, kind, cfg), out

    @staticmethod
    def backward(ctx, g_loss, _g_out):
        if g_loss is None:
            return (None, ) * 12

        def recompute():
            hidden, lm_weight, value, action, adv, weight, lp_old, lp_pre, ret = ctx.saved_tensors
            return lm_linear_pg_(hidden, lm_weight, action, adv, weight, lp_old, lp_pre, value, ret, *ctx.cfg,
                                 *ctx.needs_input_grad[:3])[1:]

        return tuple(_lm_backward(ctx, g_loss, recompute)) + (None, ) * 9


def lm_logp_fwd_(hidden, lm_weight, index, dt):
    """per-token log p(index) and logsumexp (N) fp32 of logits = hidden (N, D) @ lm_weight (V, D)^T, chunk by chunk"""
    N = hidden.shape[0]
    V = lm_weight.shape[0]
    dev = hidden.device
    rows, n = lm_chunk_plan(N, V, hidden.element_size(), sm_count(dev), False)
    lp = torch.empty(N, dtype=torch.float32, device=dev)
    lse = torch.empty(N, dtype=torch.float32, device=dev)
    with on_device(dev):
        L, st = lib(), stream_ptr()

        def launch(zc, r0):
            rc = L.b200rl_lm_linear_fwd(_LM_MODE['logp'], dt, ptr(zc), r0, zc.shape[0], rows, V, N, 1, ptr(index), None,
                                        None, None, None, 0, None, None, 0.0, 0.0, ptr(lp), ptr(lse), None, 0, None, 0,
                                        st)
            _lib.check(rc, 'b200rl_lm_linear_fwd')

        lm_chunks_(hidden, lm_weight, rows, n, launch, False, False)
    return lp, lse


def lm_logp_bwd_(hidden, lm_weight, index, lse, g, dt, want_dh, want_dw):
    """The backward of ``lm_logp_fwd_`` for the upstream gradient g (N) fp32: per chunk the logit GEMM again, the in-place
    launch dZ = g * (onehot(index) - softmax(Z)), then the gradient GEMMs.  -> (dH or None, dW or None)"""
    N = hidden.shape[0]
    V = lm_weight.shape[0]
    dev = hidden.device
    rows, n = lm_chunk_plan(N, V, hidden.element_size(), sm_count(dev), False)
    with on_device(dev):
        L, st = lib(), stream_ptr()

        def launch(zc, r0):
            rc = L.b200rl_lm_linear_bwd(dt, ptr(zc), r0, zc.shape[0], V, ptr(index), ptr(lse), ptr(g), st)
            _lib.check(rc, 'b200rl_lm_linear_bwd')

        return lm_chunks_(hidden, lm_weight, rows, n, launch, want_dh, want_dw)


class TokenLogpLinearFunction(torch.autograd.Function):
    """token_logp_linear: log p(index) (N) fp32 of logits = hidden @ lm_weight^T, differentiable w.r.t. hidden and
    lm_weight.  Saves hidden, lm_weight, index and the per-row logsumexp only; the backward recomputes each chunk's
    logits."""

    @staticmethod
    def forward(ctx, hidden, lm_weight, index, dt):
        lp, lse = lm_logp_fwd_(hidden, lm_weight, index, dt)
        ctx.save_for_backward(hidden, lm_weight, index, lse)
        ctx.dt = dt
        return lp

    @staticmethod
    def backward(ctx, g):
        hidden, lm_weight, index, lse = ctx.saved_tensors
        dh, dw = lm_logp_bwd_(hidden, lm_weight, index, lse, g.float().contiguous(), ctx.dt, *ctx.needs_input_grad[:2])
        return dh, dw, None, None
