"""Mint tests/golden/a2c_lm/*.npz from the unmodified reference's a2c_error (ding/rl_utils/a2c.py:10-44) on language-model
token rows, run on the CPU with the case's logits in their own dtype.

    python tests/golden/make_a2c_lm_golden.py

Inputs are not stored: make_case regenerates them from their seeds with torch's CPU generator.  Stored: policy, value,
entropy, a checksum of the inputs, d (policy + 0.5 * value - 0.01 * entropy) / d value, and the same / d logit (whole for
small cases, at 4096 fixed positions plus every chosen token for the long-vocabulary ones)."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import ref_loader  # noqa: E402

OUT = os.path.join(ROOT, 'tests', 'golden', 'a2c_lm')
FULL_GRAD_LIMIT = 65536
# the upstream gradients of the fixtures' backward, the 'a2c' record's defaults: policy + 0.5 * value - 0.01 * entropy
MIX = (1.0, 0.5, -0.01)

# name -> (dtype, B, S, V, weight kind, seed, logit scale, -inf logits, peaked rows)
CASES = {
    'f32_v1003_none_inf': (torch.float32, 3, 5, 1003, None, 1, 2.0, True, False),
    'f32_v1024_mask_peaked': (torch.float32, 4, 6, 1024, 'mask', 2, 1.0, False, True),
    'f32_v32771_frac_inf': (torch.float32, 1, 3, 32771, 'frac', 3, 2.0, True, False),
    'bf16_v1000_mask': (torch.bfloat16, 4, 8, 1000, 'mask', 4, 1.0, False, False),
    'bf16_v1003_frac_peaked': (torch.bfloat16, 3, 5, 1003, 'frac', 5, 2.0, False, True),
    'bf16_v32771_none_inf': (torch.bfloat16, 1, 3, 32771, None, 6, 2.0, True, False),
}


def make_inputs(B, S, V, dtype, wkind, seed, scale, neg_inf, peaked, device='cpu'):
    """dict of logit (B, S, V) in `dtype`, action, value, adv, return_ (B, S) fp32 and weight (None or (B, S)).  adv is 0
    in one row; -inf logits never at the chosen token; a peaked row has its chosen token 60 above the rest (H ~ 0) and
    another row a different token 60 above (lp ~ -60)"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, S, V, generator=g) * scale
    d = {'action': torch.randint(0, V, (B, S), generator=g), 'value': torch.randn(B, S, generator=g),
         'adv': torch.randn(B, S, generator=g), 'return_': torch.randn(B, S, generator=g), 'weight': None}
    d['adv'].view(-1)[-1] = 0.0
    if wkind == 'mask':
        w = (torch.rand(B, S, generator=g) > 0.3).float()
        w[:, 0] = 1.0
        d['weight'] = w
    elif wkind == 'frac':
        d['weight'] = torch.rand(B, S, generator=g)
    xr, act = x.view(-1, V), d['action'].view(-1)
    if neg_inf:  # a masked part of the vocabulary; never the chosen token
        cols = torch.randperm(V, generator=g)[:max(1, V // 7)]
        keep = xr.gather(-1, act.unsqueeze(-1))
        xr[:, cols] = -float('inf')
        xr.scatter_(-1, act.unsqueeze(-1), keep)
    if peaked:
        xr[0, act[0]] += 60.0
        xr[1, (act[1] + 1) % V] += 60.0
    d['logit'] = x.to(dtype)
    return {k: (v.to(device) if isinstance(v, torch.Tensor) else v) for k, v in d.items()}


def make_case(name, device='cpu'):
    dtype, B, S, V, wkind, seed, scale, neg_inf, peaked = CASES[name]
    return make_inputs(B, S, V, dtype, wkind, seed, scale, neg_inf, peaked, device)


def checksum(d):
    """float64 sums of |x| (finite entries) over the case's tensors, in name order"""
    out = []
    for k in sorted(d):
        if isinstance(d[k], torch.Tensor):
            x = d[k].double().abs()
            out.append(float(x[torch.isfinite(x)].sum()))
    return np.array(out)


def reference_call(ref, d, mix=MIX):
    """the reference on the tensors of d: (policy, value, entropy, d mix / d logit, d mix / d value)"""
    x = d['logit'].detach().clone().requires_grad_(True)
    v = d['value'].detach().clone().requires_grad_(True)
    loss = ref.a2c_error(ref.a2c_data(x, d['action'], v, d['adv'], d['return_'], d['weight']))
    (mix[0] * loss.policy_loss + mix[1] * loss.value_loss + mix[2] * loss.entropy_loss).backward()
    return loss.policy_loss.item(), loss.value_loss.item(), loss.entropy_loss.item(), x.grad, v.grad


def sample_index(d):
    B, S, V = d['logit'].shape
    fixed = np.linspace(0, B * S * V - 1, 4096).astype(np.int64)
    chosen = (np.arange(B * S) * V + d['action'].reshape(-1).numpy()).astype(np.int64)
    return np.concatenate([fixed, chosen])


def mint(name, ref):
    d = make_case(name)
    pol, val, ent, grad, gv = reference_call(ref, d)
    grad = grad.float().reshape(-1).numpy()
    out = {'policy': np.float64(pol), 'value': np.float64(val), 'entropy': np.float64(ent), 'checksum': checksum(d),
           'grad_value': gv.reshape(-1).numpy()}
    if grad.size <= FULL_GRAD_LIMIT:
        out['grad'] = grad
    else:
        idx = sample_index(d)
        out['grad_index'], out['grad_sample'] = idx, grad[idx]
    np.savez_compressed(os.path.join(OUT, name + '.npz'), **out)


if __name__ == '__main__':
    os.makedirs(OUT, exist_ok=True)
    ref = ref_loader.load()
    for n in CASES:
        mint(n, ref)
        print('minted', n)
