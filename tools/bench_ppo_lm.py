"""ppo_policy_error on language-model logits, forward + backward, on one GPU at B = 16, S = 1024, V = 32768 (the size of
the reference's GRPO / RLOO benchmark, ding/rl_utils/README.md), fp32 and bf16, with and without logit_pretrained, with
and without the entropy bonus; the backward is that of the training mix policy - 0.01 * entropy + 0.1 * kl (each where
present).  In the same run, at the same shape: GRPO (grpo_policy_error: the same three logit streams), fp32 PPO through
ops.PPOFunction (csrc/ppo.cu's warp-per-row kernel, the path fp32 calls took before csrc/vocab.cu took them) and the
reference's ppo_policy_error (oracle/ref_loader.py, on the same CUDA tensors).

Each timing is a host clock around K iterations that end in a device synchronise, after W warm-up iterations; the median
and spread over R such runs are printed as JSON lines, after one line naming the card and its power limit.  GB/s is the
traffic floor over the median time: every logit read once plus d loss / d logit_new written once, (3 + 1) * B*S*V *
sizeof(T) with logit_pretrained (and for GRPO) and (2 + 1) * B*S*V * sizeof(T) without.  A separate, untimed pass per case
counts the kernel launches of one iteration with torch.profiler.

    python tools/bench_ppo_lm.py [--iters 10] [--warmup 3] [--repeats 5] [--shape 16 1024 32768] [--no-reference]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import di_engine_b200 as b2  # noqa: E402
from di_engine_b200 import ops  # noqa: E402
from oracle import ref_loader  # noqa: E402
from tools.bench_soft_td import card, launches, timed  # noqa: E402

R = b2.rl_utils


def inputs(B, S, V, dtype, pre):
    g = torch.Generator(device='cuda').manual_seed(0)
    new = torch.randn(B, S, V, device='cuda', generator=g) * 2
    d = {'logit_old': (new + 0.1 * torch.randn(B, S, V, device='cuda', generator=g)).to(dtype),
         'logit_pretrained': (new + 0.2 * torch.randn(B, S, V, device='cuda', generator=g)).to(dtype) if pre else None,
         'action': torch.randint(0, V, (B, S), device='cuda', generator=g),
         'adv': torch.randn(B, S, device='cuda', generator=g),
         'weight': (torch.rand(B, S, device='cuda', generator=g) > 0.1).float()}
    d['logit_new'] = new.to(dtype).requires_grad_(True)
    return d


def policy_step(api, d, entropy):
    def step():
        d['logit_new'].grad = None
        data = api.ppo_policy_data(d['logit_new'], d['logit_old'], d['action'], d['adv'], d['weight'],
                                   d['logit_pretrained'])
        loss, _ = api.ppo_policy_error(data, entropy_bonus=entropy, kl_type='k3')
        total = loss.policy_loss
        if entropy:
            total = total - 0.01 * loss.entropy_loss
        if d['logit_pretrained'] is not None:
            total = total + 0.1 * loss.kl_div
        total.backward()
    return step


def old_path_step(d, entropy):
    """the same loss on csrc/ppo.cu's kernels (ops.PPOFunction, fp32 only), as fp32 calls ran before"""
    B, S, V = d['logit_new'].shape
    rows = B * S
    z = torch.zeros(rows, device='cuda')
    vn = z.clone().requires_grad_(True)
    old = d['logit_old'].reshape(rows, V)
    pre = d['logit_pretrained'].reshape(rows, V) if d['logit_pretrained'] is not None else None
    act, adv, w = d['action'].reshape(-1), d['adv'].reshape(-1), d['weight'].reshape(-1)

    def step():
        d['logit_new'].grad = None
        p, _, e, k, _ = ops.PPOFunction.apply(d['logit_new'].reshape(rows, V), vn, old, act, z, adv, z, w, pre, rows, 1,
                                              V, 0.2, 0, 0.0, 3, 'policy')
        total = p
        if entropy:
            total = total - 0.01 * e
        if pre is not None:
            total = total + 0.1 * k
        total.backward()
    return step


def grpo_step(d):
    B = d['logit_new'].shape[0]
    ref = d['logit_pretrained']
    adv = d['adv'][:, 0].contiguous()

    def step():
        d['logit_new'].grad = None
        data = R.grpo_policy_data(d['logit_new'], d['logit_old'], ref, d['action'], adv, d['weight'])
        R.grpo_policy_error(data)[0].backward()
    assert adv.numel() == B
    return step


def record(case, d, impl, step, a, floor):
    t = timed(step, a.iters, a.warmup, a.repeats)
    B, S, V = d['logit_new'].shape
    rec = {**case, 'dtype': str(d['logit_new'].dtype).replace('torch.', ''), 'shape': [B, S, V], 'impl': impl, **t,
           'floor_bytes': floor, 'gb_per_s_vs_floor': round(floor / (t['median_us'] * 1e-6) / 1e9, 1), **launches(step)}
    print(json.dumps(rec), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--repeats', type=int, default=5)
    ap.add_argument('--shape', type=int, nargs=3, default=[16, 1024, 32768])
    ap.add_argument('--no-reference', action='store_true')
    a = ap.parse_args()
    B, S, V = a.shape
    print(json.dumps(card()), flush=True)
    ref = ref_loader.load() if ref_loader.available() and not a.no_reference else None
    for dtype in (torch.float32, torch.bfloat16):
        for pre in (False, True):
            d = inputs(B, S, V, dtype, pre)
            floor = (4 if pre else 3) * B * S * V * d['logit_new'].element_size()
            for entropy in (False, True):
                case = {'case': 'ppo_policy_error', 'logit_pretrained': pre, 'entropy_bonus': entropy}
                record(case, d, 'di_engine_b200', policy_step(R, d, entropy), a, floor)
                if dtype == torch.float32:
                    record(case, d, 'ops.PPOFunction (csrc/ppo.cu)', old_path_step(d, entropy), a, floor)
                if ref is not None:
                    record(case, d, 'reference', policy_step(ref, d, entropy), a, floor)
            if pre:  # GRPO reads the same three logit tensors
                record({'case': 'grpo_policy_error'}, d, 'di_engine_b200', grpo_step(d), a, floor)
            del d
            torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
