"""a2c_error on language-model logits, forward + backward of policy + 0.5 * value - 0.01 * entropy (the 'a2c' record's
default mix), on one GPU at B = 16, S = 1024, V = 32768, fp32 and bf16.  In the same run, at the same shape: fp32 through
ops.A2CFunction (csrc/heads.cu's thread-per-row a2c_kernel, the path fp32 calls took before csrc/vocab.cu took them), the
reference's a2c_error (oracle/ref_loader.py, on the same CUDA tensors), and GRPO (grpo_policy_error, three logit streams)
for the rate of the same row kernel.

Timing, JSON lines and launch counts are tools/bench_ppo_lm.py's.  GB/s is the traffic floor over the median time:
logit read once plus d loss / d logit written once, (1 + 1) * B*S*V * sizeof(T) for A2C, (3 + 1) * B*S*V * sizeof(T) for
GRPO.  For the library's paths a separate, untimed pass also prints each kernel's device time per iteration
(torch.profiler), which splits the A2C time into the streaming launch, the loss-sum finalize and the backward launch.

    python tools/bench_a2c_lm.py [--iters 10] [--warmup 3] [--repeats 5] [--shape 16 1024 32768] [--no-reference]
"""
import argparse
import json
import os
import sys
from collections import defaultdict

import torch
from torch.profiler import ProfilerActivity, profile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import di_engine_b200 as b2  # noqa: E402
from di_engine_b200 import ops  # noqa: E402
from oracle import ref_loader  # noqa: E402
from tools.bench_ppo_lm import grpo_step, record  # noqa: E402
from tools.bench_ppo_lm import inputs as ppo_inputs  # noqa: E402
from tools.bench_soft_td import card  # noqa: E402

R = b2.rl_utils
MIX = (1.0, 0.5, -0.01)


def inputs(B, S, V, dtype):
    g = torch.Generator(device='cuda').manual_seed(0)
    d = {'logit': (torch.randn(B, S, V, device='cuda', generator=g) * 2).to(dtype).requires_grad_(True),
         'action': torch.randint(0, V, (B, S), device='cuda', generator=g),
         'value': torch.randn(B, S, device='cuda', generator=g).requires_grad_(True),
         'adv': torch.randn(B, S, device='cuda', generator=g),
         'return_': torch.randn(B, S, device='cuda', generator=g),
         'weight': (torch.rand(B, S, device='cuda', generator=g) > 0.1).float()}
    d['logit_new'] = d['logit']  # record() reads the shape and dtype from here
    return d


def a2c_step(api, d):
    def step():
        d['logit'].grad = d['value'].grad = None
        loss = api.a2c_error(api.a2c_data(d['logit'], d['action'], d['value'], d['adv'], d['return_'], d['weight']))
        (MIX[0] * loss.policy_loss + MIX[1] * loss.value_loss + MIX[2] * loss.entropy_loss).backward()
    return step


def old_path_step(d):
    """the same loss on csrc/heads.cu's a2c_kernel (ops.A2CFunction, fp32 only), as fp32 calls ran before"""
    B, S, V = d['logit'].shape
    rows = B * S
    act, adv, ret, w = (d[k].reshape(rows) for k in ('action', 'adv', 'return_', 'weight'))

    def step():
        d['logit'].grad = d['value'].grad = None
        p, vl, e = ops.A2CFunction.apply(d['logit'].reshape(rows, V), d['value'].reshape(rows), act, adv, ret, w, rows, V)
        (MIX[0] * p + MIX[1] * vl + MIX[2] * e).backward()
    return step


def kernel_times(case, impl, step):
    """device time per iteration of each kernel of one iteration (after a warm-up call), untimed by the host clock"""
    step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    us = defaultdict(float)
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            us[e.name[:90]] += e.device_time_total if hasattr(e, 'device_time_total') else e.cuda_time_total
    print(json.dumps({**case, 'impl': impl, 'kernel_us': {k: round(v, 1) for k, v in sorted(us.items(),
                                                                                         key=lambda kv: -kv[1])}}),
          flush=True)


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
        d = inputs(B, S, V, dtype)
        floor = 2 * B * S * V * d['logit'].element_size()
        case = {'case': 'a2c_error'}
        record(case, d, 'di_engine_b200', a2c_step(R, d), a, floor)
        kernel_times(case, 'di_engine_b200', a2c_step(R, d))
        if dtype == torch.float32:  # one thread per row: far slower, so fewer iterations
            slow = argparse.Namespace(iters=max(1, a.iters // 5), warmup=1, repeats=3)
            record(case, d, 'ops.A2CFunction (csrc/heads.cu)', old_path_step(d), slow, floor)
        if ref is not None:
            record(case, d, 'reference', a2c_step(ref, d), a, floor)
        del d
        torch.cuda.empty_cache()
        d = ppo_inputs(B, S, V, dtype, True)  # GRPO reads three logit tensors
        record({'case': 'grpo_policy_error'}, d, 'di_engine_b200', grpo_step(d), a, 4 * B * S * V * d['logit_new'].element_size())
        kernel_times({'case': 'grpo_policy_error'}, 'di_engine_b200', grpo_step(d))
        del d
        torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
