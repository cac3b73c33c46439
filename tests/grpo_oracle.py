"""float64 restatement of grpo_policy_error / rloo_policy_error (ding/rl_utils/grpo.py, rloo.py) and of the per-token
log-probability, plus the seeded cases of tests/golden/grpo_rloo/ (the fixtures store the reference's outputs only; the
inputs are regenerated here from their seeds with torch's CPU generator)."""
import numpy as np
import torch

CLIP, BETA = 0.2, 0.1

# name -> (loss, B, S, V, K (RLOO) or 0, dtype, weight kind, seed, logit scale)
CASES = {
    'grpo_f32_small': ('grpo', 4, 8, 1000, 0, torch.float32, None, 1, 1.0),
    'grpo_f32_mask': ('grpo', 4, 8, 1000, 0, torch.float32, 'mask', 2, 1.0),
    'grpo_f32_v2': ('grpo', 3, 5, 2, 0, torch.float32, 'mask', 3, 2.0),
    'grpo_f32_v33': ('grpo', 2, 7, 33, 0, torch.float32, None, 4, 3.0),
    'grpo_f32_v1021': ('grpo', 2, 9, 1021, 0, torch.float32, 'zero_row', 5, 4.0),
    'grpo_bf16_small': ('grpo', 4, 8, 1000, 0, torch.bfloat16, None, 6, 1.0),
    'grpo_bf16_mask': ('grpo', 4, 8, 1003, 0, torch.bfloat16, 'mask', 7, 2.0),
    'grpo_bf16_v152064': ('grpo', 1, 3, 152064, 0, torch.bfloat16, None, 8, 2.0),
    'grpo_f32_v152063': ('grpo', 1, 2, 152063, 0, torch.float32, 'mask', 9, 2.0),
    'rloo_f32_k2': ('rloo', 4, 8, 1000, 2, torch.float32, None, 11, 1.0),
    'rloo_f32_k8_mask': ('rloo', 8, 6, 517, 8, torch.float32, 'mask', 12, 2.0),
    'rloo_f32_k2_zero_row': ('rloo', 4, 5, 77, 2, torch.float32, 'zero_row', 13, 1.0),
    'rloo_bf16_k2': ('rloo', 4, 8, 1000, 2, torch.bfloat16, None, 14, 1.0),
    'rloo_bf16_k8': ('rloo', 8, 4, 2049, 8, torch.bfloat16, 'mask', 15, 3.0),
}


def make_case(name):
    """the inputs of fixture `name`, on the CPU: dict of logit_new, logit_old[, logit_ref], action, adv | reward, weight"""
    kind, B, S, V, K, dtype, wkind, seed, scale = CASES[name]
    g = torch.Generator().manual_seed(seed)
    new = torch.randn(B, S, V, generator=g) * scale
    d = {'logit_new': new, 'logit_old': new + 0.1 * torch.randn(B, S, V, generator=g)}
    if kind == 'grpo':
        d['logit_ref'] = new + 0.2 * torch.randn(B, S, V, generator=g)
        d['adv'] = torch.randn(B, generator=g)
        d['adv'][0] = 0.0  # adv = 0: both sides of the min are 0 (a tie)
    else:
        d['reward'] = torch.randn(K, B // K, generator=g)
    d['action'] = torch.randint(0, V, (B, S), generator=g)
    d['weight'] = None
    if wkind is not None:
        w = (torch.rand(B, S, generator=g) > 0.3).float()
        w[:, 0] = 1.0
        if wkind == 'zero_row':
            w[-1] = 0.0  # a sequence without any weight: the reference's loss is NaN (0 / 0)
        d['weight'] = w
    for k in ('logit_new', 'logit_old', 'logit_ref'):
        if k in d:
            d[k] = d[k].to(dtype)
    return d


def checksum(d):
    """float64 sums of |x| over the case's tensors, in name order: detects a change in how the inputs are regenerated"""
    return np.array([float(d[k].double().abs().sum()) for k in sorted(d) if isinstance(d[k], torch.Tensor)])


def logp64(logits, index, dtype=torch.float64):
    """log softmax(logits)[index] in ``dtype`` (float32: the reference's efficient_method on fp32 logits)"""
    x = logits.to(dtype)
    return x.gather(-1, index.unsqueeze(-1)).squeeze(-1) - torch.logsumexp(x, -1)


def rloo_adv64(reward, dtype=torch.float64):
    r = reward.to(dtype).reshape(reward.shape[0], -1)
    return (r - (r.sum(0) - r) / (r.shape[0] - 1)).flatten()


def head64(lp_new, lp_old, lp_ref, adv, weight, clip=CLIP, beta=BETA):
    """(loss, approx_kl, clipfrac) in the dtype of lp_new (float64 here; float32 restates the reference's own arithmetic);
    the clamp bounds are fp32(1 -+ clip), as torch forms them for fp32 ratios"""
    ratio = torch.exp(lp_new - lp_old)
    lo, hi = float(np.float32(1 - clip)), float(np.float32(1 + clip))
    a = adv.to(lp_new.dtype).reshape(-1, 1)
    tok = -torch.min(ratio * a, torch.clamp(ratio, lo, hi) * a)
    if lp_ref is not None:
        d = lp_ref - lp_new
        tok = tok + beta * (torch.exp(d) - d - 1)
    w = torch.ones_like(tok) if weight is None else weight.to(tok.dtype)
    loss = ((tok * w).sum(1) / w.sum(1)).mean()
    return loss, (lp_old - lp_new).mean().detach(), ((ratio > hi) | (ratio < lo)).to(tok.dtype).mean()


def run64(d, clip=CLIP, beta=BETA, dtype=torch.float64, lp_old=None, lp_ref=None):
    """float64 results of the case dict `d` (any device): loss, approx_kl, clipfrac, lp_new (B, S) and dlp (B, S) =
    d loss / d lp_new; d loss / d logit_new[row] = dlp[row] * (onehot - softmax) (``grad_rows64``).  ``dtype`` float32
    restates the reference's own fp32 arithmetic on the same inputs (bf16 logits widened to fp32); 'scale' stays float64.
    ``lp_old`` / ``lp_ref`` (B, S): per-token log-probabilities given instead of ``logit_old`` / ``logit_ref`` (the
    hidden-state losses' inputs), upcast to ``dtype``"""
    B = d['logit_new'].shape[0]
    lp = {k: torch.stack([logp64(d[k][b], d['action'][b], dtype) for b in range(B)])
          for k in ('logit_new', 'logit_old', 'logit_ref') if k in d}
    for k, t in (('logit_old', lp_old), ('logit_ref', lp_ref)):
        if t is not None:
            lp[k] = t.to(lp['logit_new'].device, dtype).reshape(lp['logit_new'].shape)
    lp_new = lp['logit_new'].clone().requires_grad_(True)
    adv = d['adv'] if 'adv' in d else rloo_adv64(d['reward'], dtype)
    loss, kl, cf = head64(lp_new, lp['logit_old'], lp.get('logit_ref'), adv.to(lp_new.device), d['weight'], clip,
                          beta if 'logit_ref' in lp else 0.0)
    loss.backward()
    # the size of the terms that make up dlp: gt * (|adv| * ratio [+ beta * (exp(lp_ref - lp_new) + 1)]) with
    # gt = w / (B * sum_s w).  One ulp of an fp32 logsumexp moves dlp by about that much times 2^-23 * |logsumexp|, even
    # where the terms cancel to a small dlp, so a gradient check scales its absolute bar with it
    w = torch.ones_like(lp_new) if d['weight'] is None else d['weight'].double().to(lp_new.device)
    gt = w / w.sum(1, keepdim=True) / B
    a = adv.double().to(lp_new.device).reshape(-1, 1).abs()
    lpd = {k: v.double() for k, v in lp.items()}
    scale = gt * a * torch.exp(lpd['logit_new'] - lpd['logit_old'])
    if 'logit_ref' in lp:
        scale = scale + gt * beta * (torch.exp(lpd['logit_ref'] - lpd['logit_new']) + 1)
    return {'loss': loss.item(), 'approx_kl': kl.item(), 'clipfrac': cf.item(), 'lp_new': lp['logit_new'],
            'dlp': lp_new.grad, 'scale': scale.detach()}


def grad_rows64(logits, action, dlp, dtype=torch.float64):
    """dlp[..., None] * (onehot(action) - softmax(logits)) in float64; in float32 as the reference's autograd of
    gather - logsumexp forms it, with softmax = exp(logits - logsumexp)"""
    x = logits.to(dtype)
    p = torch.softmax(x, -1) if dtype == torch.float64 else torch.exp(x - torch.logsumexp(x, -1, keepdim=True))
    g = -p * dlp.unsqueeze(-1)
    g.scatter_add_(-1, action.unsqueeze(-1), dlp.unsqueeze(-1).to(dtype))
    return g
