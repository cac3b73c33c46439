"""Mint tests/golden/grpo_rloo/*.npz from the unmodified reference (ding/rl_utils/grpo.py, rloo.py, log_prob_utils.py),
run on the CPU in the case's own dtype with its default log_prob_fn (efficient_method).

    python tests/golden/make_grpo_rloo_golden.py

Inputs are not stored: tests/grpo_oracle.make_case regenerates them from their seeds.  Stored: loss, approx_kl, clipfrac,
the per-token log-probabilities of logit_new (as float32), a checksum of the inputs, and d loss / d logit_new (whole for
small cases; at 4096 fixed positions plus every chosen token for the long-vocabulary ones)."""
import importlib
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import ref_loader  # noqa: E402
from tests import grpo_oracle  # noqa: E402

OUT = os.path.join(ROOT, 'tests', 'golden', 'grpo_rloo')
FULL_GRAD_LIMIT = 65536


def reference():
    ref_loader.load()
    return {m: importlib.import_module('ding.rl_utils.' + m) for m in ('grpo', 'rloo', 'log_prob_utils')}


def sample_index(d):
    B, S, V = d['logit_new'].shape
    n = B * S * V
    fixed = np.linspace(0, n - 1, 4096).astype(np.int64)
    chosen = (np.arange(B * S) * V + d['action'].reshape(-1).numpy()).astype(np.int64)
    return np.concatenate([fixed, chosen])


def mint(name, ref):
    d = grpo_oracle.make_case(name)
    kind = grpo_oracle.CASES[name][0]
    x = d['logit_new'].clone().requires_grad_(True)
    if kind == 'grpo':
        data = ref['grpo'].grpo_policy_data(x, d['logit_old'], d['logit_ref'], d['action'], d['adv'], d['weight'])
        loss, info = ref['grpo'].grpo_policy_error(data, clip_ratio=grpo_oracle.CLIP, beta=grpo_oracle.BETA)
    else:
        data = ref['rloo'].rloo_policy_data(x, d['logit_old'], d['action'], d['reward'], d['weight'])
        loss, info = ref['rloo'].rloo_policy_error(data, clip_ratio=grpo_oracle.CLIP)
    loss.backward()
    lp = ref['log_prob_utils'].efficient_method(d['logit_new'], d['action'])
    grad = x.grad.float().reshape(-1).numpy()
    out = {'loss': np.float64(loss.item()), 'approx_kl': np.float64(info.approx_kl),
           'clipfrac': np.float64(info.clipfrac), 'lp_new': lp.float().numpy(), 'checksum': grpo_oracle.checksum(d)}
    if grad.size <= FULL_GRAD_LIMIT:
        out['grad'] = grad
    else:
        idx = sample_index(d)
        out['grad_index'], out['grad_sample'] = idx, grad[idx]
    np.savez_compressed(os.path.join(OUT, name + '.npz'), **out)


if __name__ == '__main__':
    os.makedirs(OUT, exist_ok=True)
    ref = reference()
    for n in grpo_oracle.CASES:
        mint(n, ref)
        print('minted', n)
