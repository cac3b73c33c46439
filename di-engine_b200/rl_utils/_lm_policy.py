"""The shared body of grpo_policy_error and rloo_policy_error: argument checks, host staging, the choice between the fused
launch (a built-in log_prob_fn) and the token head on a custom log_prob_fn's output, and the info scalars."""
import torch

from .. import ops, torch_ops
from . import ppo as _ppo
from .log_prob_utils import is_fused


def check_logits(logit_new, others):
    if logit_new.dim() != 3:
        raise RuntimeError("logit_new must be (B, S, V), got %s" % (tuple(logit_new.shape), ))
    for t in others:
        if t.shape != logit_new.shape:
            raise RuntimeError("logits of one call must share a shape: %s vs %s" %
                               (tuple(logit_new.shape), tuple(t.shape)))


def check_tokens(B, S, action, weight, side):
    if tuple(action.shape) != (B, S):
        raise RuntimeError("action must be (B, S) = %s, got %s" % ((B, S), tuple(action.shape)))
    if weight is not None and tuple(weight.shape) != (B, S):
        raise RuntimeError("weight must be (B, S) = %s, got %s" % ((B, S), tuple(weight.shape)))
    if side[1].numel() != B:
        raise RuntimeError("%s must hold B = %d values, got shape %s" % (side[0], B, tuple(side[1].shape)))


def run(logits, action, weight, side, log_prob_fn, clip_ratio, beta, info_type):
    """logits: (new, old[, ref]); side: ('adv', adv) or ('reward', reward (K, B / K)).  Returns (loss, info_type)."""
    logit_new = logits[0]
    dev = ops.compute_device(*logits)
    host_out = not logit_new.is_cuda
    fused = is_fused(log_prob_fn)
    if fused:
        check_logits(logit_new, logits[1:])
        B, S, V = logit_new.shape
    else:
        # the reference's call order: new, ref, old
        lps = [log_prob_fn(logits[0], action)] + [log_prob_fn(x, action) for x in logits[:0:-1]]
        lp_new, lp_rest = lps[0], lps[1:][::-1]  # -> old[, ref]
        if lp_new.dim() != 2 or any(x.shape != lp_new.shape for x in lp_rest):
            raise RuntimeError("log_prob_fn must return (B, S) log-probabilities, got %s" %
                               ([tuple(x.shape) for x in lps], ))
        B, S = lp_new.shape
    check_tokens(B, S, action, weight, side)
    # weight / adv / reward are read as fp32 whatever their dtype (a bf16 mask or advantage included)
    w = None if weight is None else ops.to_device(weight.detach(), dev).float().contiguous()
    side_t = ops.to_device(side[1].detach(), dev).float().contiguous()
    if side[0] == 'reward':
        side_t = side_t.reshape(side_t.shape[0], -1)
    if fused:
        dt = ops.logit_dtype(*logits)
        xs = [torch_ops.stage_logits(ops.to_device(x, dev)) for x in logits]
        xs[1:] = [x.detach() for x in xs[1:]]
        a = ops.i64c(ops.to_device(action, dev), V)
        grpo = side[0] == 'adv'
        loss, kl, cf = torch_ops.lm_policy(xs[0], xs[1], xs[2] if grpo else None, a, side_t.reshape(-1) if grpo else side_t,
                                           w, 'grpo' if grpo else 'rloo', dt, clip_ratio, beta)
    else:
        lp_new = ops.to_device(lp_new, dev).float().contiguous()
        lp_rest = [ops.f32c(ops.to_device(x.detach(), dev).float()) for x in lp_rest]
        lp_ref = lp_rest[1] if len(lp_rest) > 1 else None
        adv = side_t if side[0] == 'adv' else None
        reward = side_t if side[0] == 'reward' else None
        loss, kl, cf = torch_ops.token_head(lp_new, lp_rest[0], lp_ref, adv, reward, w, clip_ratio, beta)
    if host_out:
        loss = loss.cpu()
    if torch.compiler.is_compiling():  # the host read a traced graph can take: the reference's two .item() calls
        kl, cf = kl.detach(), cf.detach()
        return loss, info_type(kl, cf) if _ppo.LAZY_INFO else info_type(kl.item(), cf.item())
    if _ppo.LAZY_INFO:
        return loss, info_type(kl, cf)
    kl, cf = torch.stack([kl, cf]).tolist()  # one host sync (the reference makes two)
    return loss, info_type(kl, cf)
