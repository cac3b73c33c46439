"""One-launch learner step: ``gae`` followed by ``ppo_error`` (csrc/fused.cu).

Not a reference function -- the reference has no fused operator -- but exactly the composition
``adv = gae(gae_data(...), gamma, lambda_); ppo_error(ppo_data(..., adv=adv.view(-1), ...), ...)`` of the two reference
signatures (ding/rl_utils/gae.py:25, ppo.py:77), which is the composite BASELINE.json measures.  Falls back to the two
separate operators when the fused kernel does not support the shapes.
"""
from typing import Optional

import torch

from .. import ops
from .gae import gae, gae_data
from .ppo import _KL_TYPES, ppo_data, ppo_error, ppo_info, ppo_loss
from . import ppo as _ppo


def gae_ppo_error(
        gae_in,
        ppo_in,
        gamma: float = 0.99,
        lambda_: float = 0.97,
        clip_ratio: float = 0.2,
        use_value_clip: bool = True,
        dual_clip: Optional[float] = None,
        kl_type: str = 'k1'
):
    """
    Arguments: ``gae_in`` a ``gae_data`` of (T, B) tensors; ``ppo_in`` a ``ppo_data`` whose ``adv`` field is ignored
    (pass None) and whose other fields cover the same T*B transitions in time-major order (logits (T*B, N) or (T, B, N)).
    Returns ``(adv, ppo_loss, ppo_info)``: adv (T, B) as ``gae`` returns it, and what ``ppo_error`` returns.
    """
    assert dual_clip is None or dual_clip > 1.0, "dual_clip value must be greater than 1.0, but get value: {}".format(
        dual_clip
    )
    value, next_value, reward, done, traj_flag = gae_in
    logit_new, logit_old, action, value_new, value_old, _adv, return_, weight, logit_pretrained = ppo_in
    if logit_pretrained is not None and kl_type not in _KL_TYPES:
        raise ValueError(f"Unknown kl_type: {kl_type}")
    if logit_new.dtype == torch.bfloat16:  # not even through the two-operator fallback
        raise TypeError(_ppo._BF16_SHAPES)

    def fallback():
        adv = gae(gae_data(value, next_value, reward, done, traj_flag), gamma, lambda_)
        data = ppo_data(logit_new, logit_old, action, value_new, value_old, adv.reshape(value_new.shape), return_,
                        weight, logit_pretrained)
        loss, info = ppo_error(data, clip_ratio, use_value_clip, dual_clip, kl_type)
        return adv, loss, info

    if value.dim() != 2 or reward.shape != value.shape or not value.is_cuda or not logit_new.is_cuda:
        return fallback()
    T, B = value.shape
    N = logit_new.shape[-1]
    if logit_new.numel() != T * B * N or value_new.numel() != T * B or action.numel() != T * B:
        return fallback()
    for name, t_, want in (('logit_old', logit_old, T * B * N), ('logit_pretrained', logit_pretrained, T * B * N),
                           ('value_old', value_old, T * B), ('return_', return_, T * B), ('next_value', next_value, T * B),
                           ('done', done, T * B), ('traj_flag', traj_flag, T * B)):
        if t_ is not None and t_.numel() != want:
            raise ValueError("gae_ppo_error: %s %s does not cover the (T=%d, B=%d) batch" % (name, tuple(t_.shape), T, B))
    f32 = ops.f32c
    v, r = f32(value.detach(), 'value'), f32(reward.detach(), 'reward')
    nv_src = next_value.detach()
    nv = f32(nv_src, 'next_value')
    d = f32(done.detach(), 'done') if done is not None else None
    tf = f32(traj_flag.detach(), 'traj_flag') if traj_flag is not None else None
    ln, lo = f32(logit_new, 'logit_new'), f32(logit_old.detach(), 'logit_old')
    lp = f32(logit_pretrained.detach(), 'logit_pretrained') if logit_pretrained is not None else None
    vn, vo = f32(value_new, 'value_new'), f32(value_old.detach(), 'value_old')
    rt = f32(return_.detach(), 'return_')
    w = f32(weight.detach(), 'weight') if weight is not None else None
    if w is not None and w.numel() != T * B:
        return fallback()
    act = ops.i64c(action, N)
    ok = ops.lib().b200rl_gae_ppo_supported(
        ops.ptr(v), ops.ptr(nv), ops.ptr(r), ops.ptr(d), ops.ptr(tf), T, B, ops.ptr(ln), ops.ptr(lo), ops.ptr(lp),
        ops.ptr(act), ops.ptr(vn), ops.ptr(vo), ops.ptr(rt), ops.ptr(w), N, ops.ptr(v), None
    )
    if not ok:
        return fallback()
    adv, p, vl, e, k, out = ops.GAEPPOFunction.apply(
        ln, vn, v, nv, r, d, tf, lo, act, vo, rt, w, lp, T, B, N, float(gamma), float(lambda_), float(clip_ratio),
        1 if use_value_clip else 0, float(dual_clip) if dual_clip is not None else 0.0, _KL_TYPES.get(kl_type, 1)
    )
    if d is not None and nv.data_ptr() != nv_src.data_ptr():
        with torch.no_grad():
            next_value.copy_(nv)
    if _ppo.LAZY_INFO:
        info = ppo_info(out[4], out[5])
    else:
        approx_kl, clipfrac = out[4:6].tolist()
        info = ppo_info(approx_kl, clipfrac)
    return adv, ppo_loss(p, vl, e, k), info
