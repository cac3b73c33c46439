"""Mint tests/golden/ppo_lm/*.npz from the unmodified reference's ppo_policy_error (ding/rl_utils/ppo.py:143-230), run on
the CPU in the case's own dtype.

    python tests/golden/make_ppo_lm_golden.py

Inputs are not stored: tests/ppo_lm_oracle.make_case regenerates them from their seeds.  Stored: policy, entropy, kl,
approx_kl, clipfrac, a checksum of the inputs, and d (policy - 0.01 * entropy + 0.1 * kl) / d logit_new (each term where
the call has it; whole for small cases, at 4096 fixed positions plus every chosen token for the long-vocabulary ones)."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import ref_loader  # noqa: E402
from tests import ppo_lm_oracle as po  # noqa: E402

OUT = os.path.join(ROOT, 'tests', 'golden', 'ppo_lm')
FULL_GRAD_LIMIT = 65536


def sample_index(d):
    B, S, V = d['logit_new'].shape
    fixed = np.linspace(0, B * S * V - 1, 4096).astype(np.int64)
    chosen = (np.arange(B * S) * V + d['action'].reshape(-1).numpy()).astype(np.int64)
    return np.concatenate([fixed, chosen])


def reference_call(ref, d, dual_clip, kl_type, entropy_bonus, mix=po.MIX):
    """the reference on the tensors of d: (policy, entropy, kl, approx_kl, clipfrac, d mix / d logit_new)"""
    x = d['logit_new'].detach().clone().requires_grad_(True)
    data = ref.ppo_policy_data(x, d['logit_old'], d['action'], d['adv'], d['weight'], d['logit_pretrained'])
    loss, info = ref.ppo_policy_error(data, clip_ratio=po.CLIP, dual_clip=dual_clip, entropy_bonus=entropy_bonus,
                                      kl_type=kl_type)
    total = mix[0] * loss.policy_loss
    if entropy_bonus:
        total = total + mix[1] * loss.entropy_loss
    if d['logit_pretrained'] is not None:
        total = total + mix[2] * loss.kl_div
    total.backward()
    return (loss.policy_loss.item(), float(loss.entropy_loss), loss.kl_div.item(), info.approx_kl, info.clipfrac,
            x.grad)


def mint(name, ref):
    d = po.make_case(name)
    pol, ent, kl, akl, cf, grad = reference_call(ref, d, *po.case_args(name))
    grad = grad.float().reshape(-1).numpy()
    out = {'policy': np.float64(pol), 'entropy': np.float64(ent), 'kl': np.float64(kl), 'approx_kl': np.float64(akl),
           'clipfrac': np.float64(cf), 'checksum': po.checksum(d)}
    if grad.size <= FULL_GRAD_LIMIT:
        out['grad'] = grad
    else:
        idx = sample_index(d)
        out['grad_index'], out['grad_sample'] = idx, grad[idx]
    np.savez_compressed(os.path.join(OUT, name + '.npz'), **out)


if __name__ == '__main__':
    os.makedirs(OUT, exist_ok=True)
    ref = ref_loader.load()
    for n in po.CASES:
        mint(n, ref)
        print('minted', n)
