"""float64 restatement of ppo_policy_error (ding/rl_utils/ppo.py:143-230, calculate_kl_div :30-54) on language-model
token rows, and the seeded cases of tests/golden/ppo_lm/ (the fixtures store the reference's outputs only; the inputs are
regenerated here from their seeds with torch's CPU generator)."""
import numpy as np
import torch

CLIP = 0.2
# the upstream gradients of the fixtures' backward: policy_loss - 0.01 * entropy_loss + 0.1 * kl_div (each where present)
MIX = (1.0, -0.01, 0.1)

# name -> (dtype, B, S, V, weight kind, dual_clip, kl_type (None: no logit_pretrained), entropy_bonus, seed, logit scale,
#          -inf logits)
CASES = {
    'f32_v1000_k1': (torch.float32, 4, 8, 1000, None, None, 'k1', True, 1, 1.0, False),
    'f32_v1003_mask_dc_k2': (torch.float32, 3, 5, 1003, 'mask', 2.0, 'k2', True, 2, 2.0, False),
    'f32_v1024_frac_k3_noent': (torch.float32, 4, 6, 1024, 'frac', None, 'k3', False, 3, 1.0, False),
    'f32_v1024_mask_dc_nopre': (torch.float32, 2, 8, 1024, 'mask', 3.0, None, True, 4, 3.0, False),
    'f32_v32771_frac_k3_inf': (torch.float32, 1, 3, 32771, 'frac', None, 'k3', True, 5, 2.0, True),
    'f32_v1003_inf_nopre_noent': (torch.float32, 2, 4, 1003, None, None, None, False, 6, 1.0, True),
    'bf16_v1000_mask_k3_noent': (torch.bfloat16, 4, 8, 1000, 'mask', None, 'k3', False, 7, 1.0, False),
    'bf16_v1003_frac_dc_k1': (torch.bfloat16, 3, 5, 1003, 'frac', 2.0, 'k1', True, 8, 2.0, False),
    'bf16_v32771_k2_inf': (torch.bfloat16, 1, 3, 32771, None, None, 'k2', True, 9, 2.0, True),
    'bf16_v1024_nopre_noent': (torch.bfloat16, 4, 4, 1024, None, None, None, False, 10, 1.0, False),
}


def make_inputs(B, S, V, dtype, wkind, kl, seed, scale, neg_inf, device='cpu'):
    """dict of logit_new, logit_old, logit_pretrained (None without KL), action, adv, weight (None or (B, S))"""
    g = torch.Generator().manual_seed(seed)
    new = torch.randn(B, S, V, generator=g) * scale
    d = {'logit_new': new, 'logit_old': new + 0.1 * torch.randn(B, S, V, generator=g),
         'logit_pretrained': new + 0.2 * torch.randn(B, S, V, generator=g) if kl else None}
    d['action'] = torch.randint(0, V, (B, S), generator=g)
    d['adv'] = torch.randn(B, S, generator=g)
    d['adv'][0, 0] = 0.0  # adv = 0: both sides of the min are 0 (a tie)
    d['weight'] = None
    if wkind == 'mask':
        w = (torch.rand(B, S, generator=g) > 0.3).float()
        w[:, 0] = 1.0
        d['weight'] = w
    elif wkind == 'frac':
        d['weight'] = torch.rand(B, S, generator=g)
    if neg_inf:  # a masked part of the vocabulary, in every logit tensor; never the chosen token
        cols = torch.randperm(V, generator=g)[:max(1, V // 7)]
        for k in ('logit_new', 'logit_old', 'logit_pretrained'):
            if d[k] is not None:
                x = d[k].clone()
                x[..., cols] = -float('inf')
                x.scatter_(-1, d['action'].unsqueeze(-1), d[k].gather(-1, d['action'].unsqueeze(-1)))
                d[k] = x
    for k in ('logit_new', 'logit_old', 'logit_pretrained'):
        if d[k] is not None:
            d[k] = d[k].to(dtype)
    return {k: (v.to(device) if isinstance(v, torch.Tensor) else v) for k, v in d.items()}


def make_case(name, device='cpu'):
    dtype, B, S, V, wkind, dual, kl, ent, seed, scale, neg_inf = CASES[name]
    return make_inputs(B, S, V, dtype, wkind, kl, seed, scale, neg_inf, device)


def case_args(name):
    """(dual_clip, kl_type, entropy_bonus) of fixture `name`"""
    c = CASES[name]
    return c[5], c[6] or 'k1', c[7]


def checksum(d):
    """float64 sums of |x| (finite entries) over the case's tensors, in name order"""
    out = []
    for k in sorted(d):
        if isinstance(d[k], torch.Tensor):
            x = d[k].double().abs()
            out.append(float(x[torch.isfinite(x)].sum()))
    return np.array(out)


def _normalized(x):
    """log softmax(x): float64 as log_softmax; float32 as Categorical(logits=x).logits forms it, x - logsumexp(x)"""
    if x.dtype == torch.float64:
        return torch.log_softmax(x, -1)
    return x - x.logsumexp(-1, keepdim=True)


def run64(d, clip=CLIP, dual_clip=None, kl_type='k1', entropy_bonus=True, mix=MIX, dtype=torch.float64, lp_old=None,
          lp_pre=None):
    """float64 results of the case dict `d` (any device): policy, entropy, kl, approx_kl, clipfrac and grad = d (mix[0] *
    policy + mix[1] * entropy + mix[2] * kl) / d logit_new, and per row lse, lp_new and H (entropy_bonus).  The clamp /
    clipfrac bounds are fp32(1 -+ clip), as torch forms them for fp32 ratios; Categorical.entropy's clamp of log p at
    finfo.min makes a -inf logit contribute 0.  ``dtype`` float32 restates the reference's own fp32 arithmetic on the same
    inputs (bf16 logits widened to fp32), the clamp at finfo(float32).min included.  ``lp_old`` / ``lp_pre`` (B, S):
    per-token log-probabilities given instead of ``logit_old`` / ``logit_pretrained`` (the hidden-state losses' inputs),
    upcast to ``dtype``."""
    x = d['logit_new'].detach().to(dtype, copy=True).requires_grad_(True)
    a = d['action'].unsqueeze(-1)
    lsm = _normalized(x)
    lp_new = lsm.gather(-1, a).squeeze(-1)
    if lp_old is None:
        lp_old = _normalized(d['logit_old'].to(dtype)).gather(-1, a).squeeze(-1)
    else:
        lp_old = lp_old.to(x.device, dtype).reshape(lp_new.shape)
    adv = d['adv'].to(dtype).reshape(lp_new.shape)
    w = torch.ones_like(adv) if d['weight'] is None else d['weight'].to(dtype).expand_as(adv)
    ratio = torch.exp(lp_new - lp_old)
    lo, hi = float(np.float32(1 - clip)), float(np.float32(1 + clip))
    sel = torch.min(ratio * adv, ratio.clamp(lo, hi) * adv)
    if dual_clip is not None:
        sel = torch.where(adv < 0, torch.max(sel, dual_clip * adv), sel)
    policy = (-sel * w).mean()
    total = mix[0] * policy
    ent = torch.zeros((), dtype=dtype)
    H = None
    if entropy_bonus:
        p = torch.exp(lsm) if dtype == torch.float64 else torch.softmax(lsm, -1)
        H = -(p * lsm.clamp(min=torch.finfo(dtype).min)).sum(-1)
        ent = (H * w).mean()
        total = total + mix[1] * ent
    kl = torch.zeros((), dtype=dtype)
    if lp_pre is not None:
        lr = lp_new - lp_pre.to(x.device, dtype).reshape(lp_new.shape)
    elif d.get('logit_pretrained') is not None:
        lr = lp_new - _normalized(d['logit_pretrained'].to(dtype)).gather(-1, a).squeeze(-1)
    if lp_pre is not None or d.get('logit_pretrained') is not None:
        kl = {'k1': lr, 'k2': lr ** 2 / 2, 'k3': torch.exp(-lr) - 1 + lr}[kl_type].mean()
        total = total + mix[2] * kl
    total.backward()
    with torch.no_grad():
        approx_kl = (lp_old - lp_new).mean()
        clipfrac = ((ratio > hi) | (ratio < lo)).to(dtype).mean()
        lse = torch.logsumexp(x, -1)
    return {'policy': policy.item(), 'entropy': ent.item(), 'kl': kl.item(), 'approx_kl': approx_kl.item(),
            'clipfrac': clipfrac.item(), 'grad': x.grad, 'lse': lse, 'lp_new': lp_new.detach(),
            'H': None if H is None else H.detach()}
