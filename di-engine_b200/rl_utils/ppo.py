"""``ppo_error`` with the signature and namedtuples of ding/rl_utils/ppo.py:8-27,77-83 -- csrc/ppo.cu; and its two halves as
the reference exposes them separately (PPG, off-policy PPO, the hybrid-action PPO): ``ppo_policy_error`` (ppo.py:143-230) and
``ppo_value_error`` (ppo.py:233-275).  The continuous-action forms ``ppo_error_continuous`` (ppo.py:278-374) and
``ppo_policy_error_continuous`` (ppo.py:377-450) run on csrc/heads.cu.  Language-model calls of ``ppo_policy_error`` /
``ppo_error`` -- one logit row per advantage, bf16 logits or fp32 with V >= ``LM_MIN_VOCAB`` -- run on the vocabulary-scale
row kernel of csrc/vocab.cu."""
from collections import namedtuple
from typing import Optional, Tuple

import torch

from .. import ops, torch_ops

ppo_data = namedtuple(
    'ppo_data',
    ['logit_new', 'logit_old', 'action', 'value_new', 'value_old', 'adv', 'return_', 'weight', 'logit_pretrained']
)
ppo_data_continuous = namedtuple(
    'ppo_data_continuous', [
        'mu_sigma_new', 'mu_sigma_old', 'action', 'value_new', 'value_old', 'adv', 'return_', 'weight',
        'logit_pretrained'
    ]
)
ppo_loss = namedtuple('ppo_loss', ['policy_loss', 'value_loss', 'entropy_loss', 'kl_div'])
ppo_info = namedtuple('ppo_info', ['approx_kl', 'clipfrac'])
ppo_policy_data = namedtuple('ppo_policy_data', ['logit_new', 'logit_old', 'action', 'adv', 'weight', 'logit_pretrained'])
ppo_policy_data_continuous = namedtuple(
    'ppo_policy_data_continuous', ['mu_sigma_new', 'mu_sigma_old', 'action', 'adv', 'weight', 'logit_pretrained']
)
ppo_policy_loss = namedtuple('ppo_policy_loss', ['policy_loss', 'entropy_loss', 'kl_div'])
ppo_value_data = namedtuple('ppo_value_data', ['value_new', 'value_old', 'return_', 'weight'])

_KL_TYPES = {'k1': 1, 'k2': 2, 'k3': 3}

# When True ``ppo_info`` carries 0-dim device tensors instead of python floats, so a training step never blocks on
# the host (the reference's two ``.item()`` calls, ppo.py:218-220, are the only host syncs of its PPO loss).
LAZY_INFO = False

# fp32 logits with at least this many classes per row (and one row per advantage) run on the vocabulary-scale row kernel
# (csrc/vocab.cu: 16-byte loads, one pass over each logit tensor) instead of csrc/ppo.cu's warp-per-row kernel, which was
# written for action spaces of ~100; bf16 logits always do, no other PPO kernel reads them
LM_MIN_VOCAB = 1024
_BF16_SHAPES = ("di_engine_b200: bfloat16 logits are taken by ppo_policy_error and ppo_error with one logit row per "
                "advantage -- logits (..., V) against action / adv / weight (...), e.g. (B, S, V) against (B, S) -- and "
                "no advantage normalisation; every other PPO call needs float32 logits")


def shape_fn_ppo(args, kwargs):
    """Plugin-cache key of the reference boundary (ding/rl_utils/ppo.py:57-68): the shape of ``logit_new``."""
    data = args[0] if len(args) > 0 else kwargs['data']
    return data.logit_new.shape


def normalize_advantage(adv: torch.Tensor) -> torch.Tensor:
    """``(adv - adv.mean()) / (adv.std() + 1e-8)`` -- PPOPolicy's per-train-batch advantage normalisation
    (ding/policy/ppo.py:304-306) as two small launches (statistics; elementwise).  ``ppo_error(..., adv_norm=True)`` applies
    the same normalisation inside the loss kernels without materialising the tensor."""
    dev = ops.compute_device(adv)
    host_out = not adv.is_cuda
    a = ops.f32c(ops.to_device(adv.detach(), dev), 'adv')
    out = torch_ops.normalize(a, torch_ops.adv_stats(a))
    return out.cpu() if host_out else out


def ppo_error(
        data: namedtuple,
        clip_ratio: float = 0.2,
        use_value_clip: bool = True,
        dual_clip: Optional[float] = None,
        kl_type: str = 'k1'
) -> Tuple[namedtuple, namedtuple]:
    """
    PPO loss (clipped surrogate with optional dual clip, clipped value loss, entropy, optional KL to a pretrained
    policy), drop-in for ding/rl_utils/ppo.py:77-140 (policy part :143-230, value part :233-275).

    Shapes: logit_new / logit_old / logit_pretrained (..., N); action (...); value_new, value_old, adv, return_,
    weight (...) -- or, multi-agent (ppo.py:199-200,:206-207), logits (B, A, N), action (B, A) with (B,) value/adv.
    Returns ``(ppo_loss, ppo_info)``: four differentiable 0-dim tensors (gradients reach ``logit_new`` and
    ``value_new``) and two python floats.

    Language-model shapes (one logit row per advantage, bf16 logits or fp32 with V >= ``LM_MIN_VOCAB``) run as the
    reference composes them: ``ppo_policy_error`` on csrc/vocab.cu plus ``ppo_value_error``.
    """
    if _lm_path(data[0], data[5]):
        logit_new, logit_old, action, value_new, value_old, adv, return_, weight, logit_pretrained = data
        policy, info = _ppo_lm(ppo_policy_data(logit_new, logit_old, action, adv, weight, logit_pretrained), clip_ratio,
                               dual_clip, True, kl_type, 'ppo')
        value_loss = ppo_value_error(ppo_value_data(value_new, value_old, return_, weight), clip_ratio, use_value_clip)
        return ppo_loss(policy.policy_loss, value_loss, policy.entropy_loss, policy.kl_div), info
    return _ppo_error(data, clip_ratio, use_value_clip, dual_clip, kl_type, 'ppo')


def ppo_error_adv_norm(
        data: namedtuple,
        clip_ratio: float = 0.2,
        use_value_clip: bool = True,
        dual_clip: Optional[float] = None,
        kl_type: str = 'k1',
        adv_stats: Optional[torch.Tensor] = None
) -> Tuple[namedtuple, namedtuple]:
    """
    ``ppo_error`` evaluated on ``(adv - adv.mean()) / (adv.std() + 1e-8)`` -- the normalisation PPOPolicy applies to every
    train batch right before the call (ding/policy/ppo.py:304-306; not a reference function, exactly those lines + ppo_error).
    One small statistics launch -- none when ``adv_stats`` (two device floats {mean, std + 1e-8}, e.g. ``gae_returns(...).adv_stats``
    for a batch that is one minibatch) is handed in; the normalisation itself happens on load inside the loss kernels (no
    normalised copy of ``adv`` is written).  Same arguments and results as ``ppo_error``.
    """
    return _ppo_error(data, clip_ratio, use_value_clip, dual_clip, kl_type, 'ppo', True, adv_stats)


def _ppo_error(data, clip_ratio, use_value_clip, dual_clip, kl_type, _hint_kind, adv_norm=False, adv_stats=None, factor=None):
    assert dual_clip is None or dual_clip > 1.0, "dual_clip value must be greater than 1.0, but get value: {}".format(
        dual_clip
    )
    logit_new, logit_old, action, value_new, value_old, adv, return_, weight, logit_pretrained = data
    if logit_pretrained is not None and kl_type not in _KL_TYPES:
        raise ValueError(f"Unknown kl_type: {kl_type}")
    if logit_new.dtype == torch.bfloat16:
        raise TypeError(_BF16_SHAPES)
    dev = ops.compute_device(logit_new, value_new, logit_old)
    host_out = not logit_new.is_cuda
    N = logit_new.shape[-1]
    rows = logit_new.numel() // N
    S = adv.numel()
    if S == 0 or rows % S != 0 or action.numel() != rows:
        raise ValueError(
            "ppo_error: logit %s / action %s / adv %s shapes do not match" %
            (tuple(logit_new.shape), tuple(action.shape), tuple(adv.shape))
        )
    G = rows // S
    if G > 1 and not (logit_new.dim() == adv.dim() + 2 and logit_new.shape[adv.dim()] == G):
        raise ValueError("ppo_error: multi-agent logits must be (B, A, N) against (B,) adv")
    # raw pointers go to the kernels: every operand must cover exactly the rows / samples the sizes above promise
    for name, t_, want in (('logit_old', logit_old, rows * N), ('logit_pretrained', logit_pretrained, rows * N),
                           ('value_new', value_new, S), ('value_old', value_old, S), ('return_', return_, S)):
        if t_ is not None and t_.numel() != want:
            raise ValueError("ppo_error: %s %s does not match logit_new %s / adv %s" %
                             (name, tuple(t_.shape), tuple(logit_new.shape), tuple(adv.shape)))

    def stage(t, name):
        return ops.f32c(ops.to_device(t, dev), name) if t is not None else None

    ln, lo, lp = stage(logit_new, 'logit_new'), stage(logit_old.detach(), 'logit_old'), None
    if logit_pretrained is not None:
        lp = stage(logit_pretrained.detach(), 'logit_pretrained')
    vn = stage(value_new, 'value_new')
    vo, ad, rt = stage(value_old.detach(), 'value_old'), stage(adv.detach(), 'adv'), stage(return_.detach(), 'return_')
    w = None
    if weight is not None:
        w = stage(weight.detach(), 'weight')
        if w.numel() != S:
            w = w.expand_as(ad).contiguous()
    act = ops.i64c(ops.to_device(action, dev), N)
    stats = None
    if adv_norm:
        if adv_stats is None:
            stats = torch_ops.adv_stats(ad)
        else:
            stats = ops.f32c(ops.to_device(adv_stats.detach(), ad.device), 'adv_stats').reshape(-1)
            if stats.numel() != 2:
                raise ValueError("adv_stats must hold two floats {mean, std + 1e-8}")
    fac = None
    if factor is not None:  # happo_error: (B, 1) -> squeeze(1) -> one factor per sample (happo.py:124-125)
        fac = stage(factor.detach(), 'factor').reshape(-1)
        if fac.numel() != S:
            raise ValueError("happo_error: factor %s does not match adv %s" % (tuple(factor.shape), tuple(adv.shape)))
    args = (ln, vn, lo, act, vo, ad, rt, w, lp, S, G, N, float(clip_ratio), 1 if use_value_clip else 0,
            float(dual_clip) if dual_clip is not None else 0.0, _KL_TYPES.get(kl_type, 1), _hint_kind, stats, fac)
    p, v, e, k, out = torch_ops.ppo(*args)
    if torch.compiler.is_compiling():  # the host read a traced graph can take: the reference's two .item() (ppo.py:218-220)
        info = ppo_info(out[4].detach(), out[5].detach()) if LAZY_INFO else ppo_info(out[4].item(), out[5].item())
    elif LAZY_INFO:
        info = ppo_info(out[4], out[5])
    else:
        approx_kl, clipfrac = out[4:6].tolist()  # one D2H read for both monitors (reference: two .item() syncs)
        info = ppo_info(approx_kl, clipfrac)
    if host_out:
        p, v, e, k = p.cpu(), v.cpu(), e.cpu(), k.cpu()
    return ppo_loss(p, v, e, k), info


def ppo_error_continuous(
        data: namedtuple,
        clip_ratio: float = 0.2,
        use_value_clip: bool = True,
        dual_clip: Optional[float] = None,
        kl_type: str = 'k1'
) -> Tuple[namedtuple, namedtuple]:
    """
    PPO loss for a continuous action space, drop-in for ding/rl_utils/ppo.py:278-374: the policies are
    ``Independent(Normal(mu, sigma), 1)`` given as dicts ``{'mu': (B, D), 'sigma': (B, D)}`` in the ``logit_new`` / ``logit_old``
    / ``logit_pretrained`` fields of ``ppo_data`` (a 1-D old policy is one action dim, ppo.py:336-337); action (B, D) float.
    Returns ``(ppo_loss, ppo_info)``; gradients reach ``mu``, ``sigma`` of the new policy and ``value_new``.  Forward and
    gradients in one launch (csrc/heads.cu), device-verified backward.
    """
    return _ppo_error_continuous(data, clip_ratio, use_value_clip, dual_clip, kl_type, 'ppoc')


def _ppo_error_continuous(data, clip_ratio, use_value_clip, dual_clip, kl_type, hint_kind, factor=None):
    """``hint_kind``: the call site's expected-upstream-gradient record (a key of ops._HINT_INIT)"""
    assert dual_clip is None or dual_clip > 1.0, "dual_clip value must be greater than 1.0, but get value: {}".format(
        dual_clip
    )
    mu_sigma_new, mu_sigma_old, action, value_new, value_old, adv, return_, weight, logit_pretrained = data
    if logit_pretrained is not None and kl_type not in _KL_TYPES:
        raise ValueError(f"Unknown kl_type: {kl_type}")
    mu, sigma = mu_sigma_new['mu'], mu_sigma_new['sigma']
    dev = ops.compute_device(mu, value_new)
    host_out = not mu.is_cuda
    S = adv.numel()
    D = mu.numel() // S

    def stage(t, name, n):
        t = ops.f32c(ops.to_device(t, dev), name)
        if t.numel() != n:
            raise ValueError("ppo_error_continuous: %s %s does not match adv %s / action dims %d" %
                             (name, tuple(t.shape), tuple(adv.shape), D))
        return t

    mo, so = mu_sigma_old['mu'].detach(), mu_sigma_old['sigma'].detach()
    args = [stage(mu, 'mu', S * D), stage(sigma, 'sigma', S * D), stage(value_new, 'value_new', S), stage(mo, 'mu_old', S * D),
            stage(so, 'sigma_old', S * D)]
    if logit_pretrained is not None:
        args += [stage(logit_pretrained['mu'].detach(), 'mu_pretrained', S * D),
                 stage(logit_pretrained['sigma'].detach(), 'sigma_pretrained', S * D)]
    else:
        args += [None, None]
    args += [stage(action.detach(), 'action', S * D), stage(value_old.detach(), 'value_old', S), stage(adv.detach(), 'adv', S),
             stage(return_.detach(), 'return_', S),
             stage(weight.detach(), 'weight', S) if weight is not None else None]
    fac = stage(factor.detach(), 'factor', S).reshape(-1) if factor is not None else None
    args += [S, D, float(clip_ratio), 1 if use_value_clip else 0, float(dual_clip) if dual_clip is not None else 0.0,
             _KL_TYPES.get(kl_type, 1), hint_kind, fac]
    p, v, e, k, out = torch_ops.ppo_continuous(*args)
    if torch.compiler.is_compiling():  # the host read a traced graph can take: the reference's two .item() (ppo.py:366-368)
        info = ppo_info(out[4].detach(), out[5].detach()) if LAZY_INFO else ppo_info(out[4].item(), out[5].item())
    elif LAZY_INFO:
        info = ppo_info(out[4], out[5])
    else:
        approx_kl, clipfrac = out[4:6].tolist()
        info = ppo_info(approx_kl, clipfrac)
    if host_out:
        p, v, e, k = p.cpu(), v.cpu(), e.cpu(), k.cpu()
    return ppo_loss(p, v, e, k), info


def ppo_policy_error(
        data: namedtuple,
        clip_ratio: float = 0.2,
        dual_clip: Optional[float] = None,
        entropy_bonus: bool = True,
        kl_type: str = 'k1'
) -> Tuple[namedtuple, namedtuple]:
    """
    Policy half of the PPO loss, drop-in for ding/rl_utils/ppo.py:143-230: ``(ppo_policy_loss(policy_loss, entropy_loss,
    kl_div), ppo_info)``.  Runs on the ``ppo_error`` kernel with a zero value head (value_new = value_old = return_ = 0
    contributes nothing and receives no gradient); its expected-upstream-gradient record is kept apart from
    ``ppo_error``'s, so alternating the two never forces a recomputation.  Language-model shapes -- logits (..., V) with
    one row per advantage, e.g. (B, S, V) against (B, S) adv / action / weight, in bf16 or in fp32 with
    V >= ``LM_MIN_VOCAB`` -- run on the vocabulary-scale row kernel of csrc/vocab.cu.
    """
    if _lm_path(data[0], data[3]):
        return _ppo_lm(data, clip_ratio, dual_clip, entropy_bonus, kl_type, 'policy')
    logit_new, logit_old, action, adv, weight, logit_pretrained = data
    zero = torch.zeros_like(adv)
    loss, info = _ppo_error(
        ppo_data(logit_new, logit_old, action, zero, zero, adv, zero, weight, logit_pretrained), clip_ratio, False,
        dual_clip, kl_type, 'policy'
    )
    entropy = loss.entropy_loss if entropy_bonus else torch.tensor(0.0)  # ppo.py:203
    return ppo_policy_loss(loss.policy_loss, entropy, loss.kl_div), info


def _lm_path(logit_new, adv):
    """whether a ppo_policy_error / ppo_error call runs on csrc/vocab.cu: one logit row per advantage, and bf16 logits or
    fp32 with V >= LM_MIN_VOCAB"""
    if logit_new.dtype not in (torch.float32, torch.bfloat16) or logit_new.dim() < 1 or logit_new.shape[-1] == 0:
        return False
    V = logit_new.shape[-1]
    return adv.numel() == logit_new.numel() // V and (logit_new.dtype == torch.bfloat16 or V >= LM_MIN_VOCAB)


def _ppo_lm(data, clip_ratio, dual_clip, entropy_bonus, kl_type, hint_kind):
    """ppo_policy_error on token rows (csrc/vocab.cu, ops.PPOLMFunction): the reference's plain means over all rows;
    ``hint_kind`` is the call site's expected-upstream-gradient record, of which the policy, entropy and kl slots are read"""
    assert dual_clip is None or dual_clip > 1.0, "dual_clip value must be greater than 1.0, but get value: {}".format(
        dual_clip
    )
    logit_new, logit_old, action, adv, weight, logit_pretrained = data
    if logit_pretrained is not None and kl_type not in _KL_TYPES:
        raise ValueError(f"Unknown kl_type: {kl_type}")
    logits = [logit_new, logit_old] + ([logit_pretrained] if logit_pretrained is not None else [])
    dt = ops.logit_dtype(*logits)
    V = logit_new.shape[-1]
    rows = logit_new.numel() // V
    for name, t_ in (('logit_old', logit_old), ('logit_pretrained', logit_pretrained), ('action', action)):
        if t_ is not None and t_.numel() != (rows if name == 'action' else rows * V):
            raise ValueError("ppo_policy_error: %s %s does not match logit_new %s" %
                             (name, tuple(t_.shape), tuple(logit_new.shape)))
    dev = ops.compute_device(*logits)
    host_out = not logit_new.is_cuda
    # logit_old / logit_pretrained get no gradient; weight and adv are read as fp32 whatever their dtype
    xs = [torch_ops.stage_logits(ops.to_device(x, dev)) for x in logits]
    xs[1:] = [x.detach() for x in xs[1:]]
    ad = ops.to_device(adv.detach(), dev).float().contiguous()
    w = None
    if weight is not None:
        w = ops.to_device(weight.detach(), dev).float()
        w = (w if w.numel() == rows else w.expand_as(ad)).contiguous()
    act = ops.i64c(ops.to_device(action, dev), V)
    args = (xs[0], xs[1], xs[2] if len(xs) > 2 else None, act, ad, w)
    cfg = (float(clip_ratio), float(dual_clip) if dual_clip is not None else 0.0, _KL_TYPES.get(kl_type, 1),
           bool(entropy_bonus))
    p, e, k, out = torch_ops.ppo_lm(*args, dt, *cfg, hint_kind)
    if torch.compiler.is_compiling():  # the host read a traced graph can take: the reference's two .item() (ppo.py:218-220)
        info = ppo_info(out[3].detach(), out[4].detach()) if LAZY_INFO else ppo_info(out[3].item(), out[4].item())
    elif LAZY_INFO:
        info = ppo_info(out[3], out[4])
    else:
        approx_kl, clipfrac = out[3:5].tolist()
        info = ppo_info(approx_kl, clipfrac)
    if host_out:
        p, e, k = p.cpu(), e.cpu(), k.cpu()
    entropy = e if entropy_bonus else torch.tensor(0.0)  # ppo.py:203
    return ppo_policy_loss(p, entropy, k), info


def ppo_policy_error_continuous(
        data: namedtuple,
        clip_ratio: float = 0.2,
        dual_clip: Optional[float] = None,
        kl_type: str = 'k1'
) -> Tuple[namedtuple, namedtuple]:
    """
    Policy half of the continuous-action PPO loss, drop-in for ding/rl_utils/ppo.py:377-450: six fields ``(mu_sigma_new,
    mu_sigma_old, action, adv, weight, logit_pretrained)`` (``ppo_policy_data_continuous``, or ``ppo_policy_data`` as
    PPOPGPolicy and PPOOffPolicy pass it), the policies dicts ``{'mu': (B, D), 'sigma': (B, D)}``, action (B, D) float.
    Returns ``(ppo_policy_loss(policy_loss, entropy_loss, kl_div), ppo_info)``; ``kl_div`` is the python int ``0`` without a
    pretrained policy, as in the reference.  Runs on the ``ppo_error_continuous`` kernel with a zero value head; its
    expected-upstream-gradient record is kept apart from ``ppo_error_continuous``'s.
    """
    mu_sigma_new, mu_sigma_old, action, adv, weight, logit_pretrained = data
    zero = torch.zeros_like(adv)
    loss, info = _ppo_error_continuous(
        ppo_data(mu_sigma_new, mu_sigma_old, action, zero, zero, adv, zero, weight, logit_pretrained), clip_ratio, False,
        dual_clip, kl_type, 'ppoc_policy'
    )
    kl_div = loss.kl_div if logit_pretrained is not None else 0  # ppo.py:448
    return ppo_policy_loss(loss.policy_loss, loss.entropy_loss, kl_div), info


def ppo_value_error(
        data: namedtuple,
        clip_ratio: float = 0.2,
        use_value_clip: bool = True,
) -> torch.Tensor:
    """
    Value half of the PPO loss, drop-in for ding/rl_utils/ppo.py:233-275: ``0.5 * mean(w * max((R - v)^2, (R - v_clip)^2))``
    (or the unclipped form); differentiable w.r.t. ``value_new``.  One small kernel (csrc/ppo.cu: ppo_value_kernel).
    """
    value_new, value_old, return_, weight = data
    dev = ops.compute_device(value_new)
    host_out = not value_new.is_cuda
    vn = ops.f32c(ops.to_device(value_new, dev), 'value_new')
    vo = ops.f32c(ops.to_device(value_old.detach(), dev), 'value_old')
    rt = ops.f32c(ops.to_device(return_.detach(), dev), 'return_')
    if vo.numel() != vn.numel() or rt.numel() != vn.numel():
        raise ValueError("ppo_value_error: value_new %s / value_old %s / return_ %s shapes do not match" %
                         (tuple(value_new.shape), tuple(value_old.shape), tuple(return_.shape)))
    w = None
    if weight is not None:
        w = ops.f32c(ops.to_device(weight.detach(), dev), 'weight')
        if w.numel() != vn.numel():
            w = w.expand_as(vn).contiguous()
    loss = torch_ops.ppo_value(vn, vo, rt, w, clip_ratio, use_value_clip)
    return loss.cpu() if host_out else loss
