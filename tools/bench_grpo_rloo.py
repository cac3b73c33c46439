"""grpo_policy_error and rloo_policy_error, forward + backward, on one GPU at the size of the reference's own benchmark
(ding/rl_utils/README.md: B = 16, S = 1024, V = 32768), fp32 and bf16 logits: the reference functions with their default
``efficient_method`` (oracle/ref_lm.py: the reference tree, or the archive build() made from it; run on CUDA tensors)
against di_engine_b200 (csrc/vocab.cu).

Each timing is a host clock around K iterations that end in a device synchronise, after W warm-up iterations; the median
and spread over R such runs are printed as JSON lines, after one line naming the card and its power limit.  GB/s is the
traffic floor over the median time: every logit read once plus d loss / d logit_new written once, (3 + 1) * B*S*V *
sizeof(T) for GRPO and (2 + 1) * B*S*V * sizeof(T) for RLOO.  A separate, untimed pass per case counts the kernel launches
of one iteration with torch.profiler.

    python tools/bench_grpo_rloo.py [--iters 20] [--warmup 3] [--repeats 5] [--shape 16 1024 32768]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import di_engine_b200 as b2  # noqa: E402
from oracle import ref_lm  # noqa: E402
from tools.bench_soft_td import card, launches, timed  # noqa: E402


def reference_loss(ref, kind, d):
    if kind == 'grpo':
        data = ref['grpo'].grpo_policy_data(d['logit_new'], d['logit_old'], d['logit_ref'], d['action'], d['adv'], d['weight'])
        return ref['grpo'].grpo_policy_error(data)[0]
    data = ref['rloo'].rloo_policy_data(d['logit_new'], d['logit_old'], d['action'], d['reward'], d['weight'])
    return ref['rloo'].rloo_policy_error(data)[0]


def ours_loss(_ref, kind, d):
    if kind == 'grpo':
        data = b2.rl_utils.grpo_policy_data(d['logit_new'], d['logit_old'], d['logit_ref'], d['action'], d['adv'], d['weight'])
        return b2.rl_utils.grpo_policy_error(data)[0]
    data = b2.rl_utils.rloo_policy_data(d['logit_new'], d['logit_old'], d['action'], d['reward'], d['weight'])
    return b2.rl_utils.rloo_policy_error(data)[0]


def inputs(kind, B, S, V, dtype):
    g = torch.Generator(device='cuda').manual_seed(0)
    new = (torch.randn(B, S, V, device='cuda', generator=g) * 2).to(dtype)
    d = {'logit_new': new.requires_grad_(True),
         'logit_old': (new.detach().float() + 0.1 * torch.randn(B, S, V, device='cuda', generator=g)).to(dtype),
         'action': torch.randint(0, V, (B, S), device='cuda', generator=g),
         'weight': (torch.rand(B, S, device='cuda', generator=g) > 0.1).float()}
    if kind == 'grpo':
        d['logit_ref'] = (new.detach().float() + 0.2 * torch.randn(B, S, V, device='cuda', generator=g)).to(dtype)
        d['adv'] = torch.randn(B, device='cuda', generator=g)
    else:
        d['reward'] = torch.randn(4, B // 4, device='cuda', generator=g)
    return d


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--repeats', type=int, default=5)
    ap.add_argument('--shape', type=int, nargs=3, default=[16, 1024, 32768])
    a = ap.parse_args()
    B, S, V = a.shape
    print(json.dumps(card()))
    with ref_lm.modules() as ref:
        run(ref, B, S, V, a)


def run(ref, B, S, V, a):
    for kind in ('grpo', 'rloo'):
        for dtype in (torch.float32, torch.bfloat16):
            d = inputs(kind, B, S, V, dtype)
            floor = (4 if kind == 'grpo' else 3) * B * S * V * d['logit_new'].element_size()
            for impl, fn in (('reference', reference_loss), ('di_engine_b200', ours_loss)):

                def step():
                    d['logit_new'].grad = None
                    fn(ref, kind, d).backward()

                t = timed(step, a.iters, a.warmup, a.repeats)
                rec = {'case': kind, 'dtype': str(dtype).replace('torch.', ''), 'shape': [B, S, V], 'impl': impl, **t,
                       'floor_bytes': floor, 'gb_per_s_vs_floor': round(floor / (t['median_us'] * 1e-6) / 1e9, 1),
                       **launches(step)}
                print(json.dumps(rec), flush=True)
            del d
            torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
