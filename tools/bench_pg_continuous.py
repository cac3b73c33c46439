"""The continuous-action policy-gradient losses, forward + backward, on one GPU: the reference functions (oracle/_ref, run on
CUDA tensors) against di_engine_b200, at the sizes of the shipped configs.

  A2C      a2c_error_continuous          B = 32,  D = 1 (dizoo/classic_control/pendulum/config/pendulum_a2c_config.py)
                                         B = 256, D = 4 (dizoo/box2d/bipedalwalker/config/bipedalwalker_a2c_config.py)
  PPOPG    ppo_policy_error_continuous   B = 64,  D = 4 (dizoo/box2d/bipedalwalker/config/bipedalwalker_ppopg_config.py)
  hybrid   ppo_policy_error_continuous   B = 320, D = 2, the continuous part of a hybrid action
                                         (dizoo/gym_hybrid/config/gym_hybrid_hppo_config.py: batch_size 320, action_args_shape 2;
                                         no shipped config selects PPOOffPolicy with a hybrid action, so this is its shape)

Each timing is a host clock around K iterations that end in a device synchronise, after W warm-up iterations; the median
and spread over R such runs are printed as JSON lines, after one line naming the card and its power limit.  A separate,
untimed pass per case counts the kernel launches of one iteration with torch.profiler.

    python tools/bench_pg_continuous.py [--iters 500] [--warmup 50] [--repeats 7]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import di_engine_b200 as b2  # noqa: E402
from oracle import ref_loader  # noqa: E402
from tools.bench_soft_td import card, launches, timed  # noqa: E402


def a2c_step(api, B, D, seed):
    """policy/a2c.py:172-182: the loss, its weighted total and the backward pass"""
    g = torch.Generator().manual_seed(seed)
    mu = torch.randn(B, D, generator=g).cuda().requires_grad_(True)
    sigma = torch.exp(0.3 * torch.randn(B, D, generator=g)).cuda().requires_grad_(True)
    value = torch.randn(B, generator=g).cuda().requires_grad_(True)
    action = mu.detach() + sigma.detach() * torch.randn(B, D, generator=g).cuda()
    adv, return_ = torch.randn(B, generator=g).cuda(), torch.randn(B, generator=g).cuda()

    def step():
        mu.grad = sigma.grad = value.grad = None
        loss = api.a2c_error_continuous(api.a2c_data({'mu': mu, 'sigma': sigma}, action, value, adv, return_, None))
        (loss.policy_loss + 0.5 * loss.value_loss - 0.01 * loss.entropy_loss).backward()
    return step


def ppo_policy_step(api, B, D, seed):
    """policy/ppo.py:796-802: the policy loss, its weighted total and the backward pass"""
    g = torch.Generator().manual_seed(seed)
    mu = torch.randn(B, D, generator=g).cuda().requires_grad_(True)
    sigma = torch.exp(0.3 * torch.randn(B, D, generator=g)).cuda().requires_grad_(True)
    old = {'mu': mu.detach() + 0.3 * torch.randn(B, D, generator=g).cuda(),
           'sigma': sigma.detach() * torch.exp(0.2 * torch.randn(B, D, generator=g)).cuda()}
    action = mu.detach() + sigma.detach() * torch.randn(B, D, generator=g).cuda()
    adv = torch.randn(B, generator=g).cuda()

    def step():
        mu.grad = sigma.grad = None
        loss, info = api.ppo_policy_error_continuous(
            api.ppo_policy_data({'mu': mu, 'sigma': sigma}, old, action, adv, None, None), 0.2)
        (loss.policy_loss - 0.01 * loss.entropy_loss).backward()
    return step


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=500)
    ap.add_argument('--warmup', type=int, default=50)
    ap.add_argument('--repeats', type=int, default=7)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_pg_continuous: needs a CUDA device")
    ref = ref_loader.load()
    print(json.dumps(card()))
    cases = [('a2c_error_continuous B=32 D=1 (Pendulum A2C)', a2c_step, 32, 1),
             ('a2c_error_continuous B=256 D=4 (BipedalWalker A2C)', a2c_step, 256, 4),
             ('ppo_policy_error_continuous B=64 D=4 (BipedalWalker PPOPG)', ppo_policy_step, 64, 4),
             ('ppo_policy_error_continuous B=320 D=2 (hybrid action, continuous part)', ppo_policy_step, 320, 2)]
    for name, make, B, D in cases:
        for impl, api in (('reference', ref), ('b200', b2.rl_utils)):
            step = make(api, B, D, 0)
            res = timed(step, args.iters, args.warmup, args.repeats)
            print(json.dumps(dict(case=name, impl=impl, **res, **launches(step))))


if __name__ == '__main__':
    main()
