"""The hidden-state losses (rl_utils/lm_linear.py) eager against ``torch.compile(fullgraph=True)``, on one GPU.  Two arms,
alternated within each repeat on the same card:

  eager     the loss as it runs without compile (in-place scale of the forward-written dH / dW in the backward)
  compiled  the same call under torch.compile (inductor, fullgraph=True): one b200rl custom op per call, whose backward
            op scales the forward-written dH / dW out of place

Workloads and calls are tools/bench_lm_linear.py's: 16 x 1024 tokens at Qwen2-7B's lm_head (D = 3584, V = 152 064,
bf16) and D = 4096, V = 32 768 in bf16 and fp32; GRPO (beta 0.1), PPO (k3 KL 0.1, entropy 0.01) and A2C (value 0.5,
entropy 0.01), each forward + backward with gradients to hidden and lm_weight (and A2C's value).  The monitors stay on
the device (ppo.LAZY_INFO) in both arms.  Printed as JSON lines after one line naming the card and its power limit:

  ms        device time from CUDA events around one forward + backward, median (min, max) of --repeats, with the arms alternated
  peak_gb   torch.cuda.max_memory_allocated during the call, above what was allocated before it (the inputs)
  compiled_minus_eager_ms   the paired difference of the two arms within each repeat: median, quartiles, min, max
  kernels   CUDA kernels in one call, from a separate torch.profiler run (GEMMs, the library's launches, torch's own),
            and kernel_names: each kernel's name (first 80 characters) and its launches in that call

    python tools/bench_compile_lm_linear.py [--repeats 30] [--warmup 2] [--losses grpo ppo a2c] [--workloads ...]
"""
import argparse
import collections
import json
import os
import sys

import torch
from torch.profiler import ProfilerActivity, profile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import di_engine_b200 as b2  # noqa: E402
from tools.bench_lm_linear import EW, KW, VW, WORKLOADS, clear, event_ms, inputs, peak_gb, summary  # noqa: E402
from tools.bench_soft_td import card  # noqa: E402

R = b2.rl_utils


def grpo(d):
    loss, _ = R.grpo_policy_error_linear(R.grpo_linear_data(d['hidden'], d['lm_weight'], d['logp_old'], d['logp_ref'],
                                                            d['action'], d['adv'], d['weight']), beta=0.1)
    return loss


def ppo(d):
    out, _ = R.ppo_policy_error_linear(R.ppo_policy_linear_data(d['hidden'], d['lm_weight'], d['logp_old'], d['action'],
                                                                d['adv_tok'], d['weight'], d['logp_ref']),
                                       kl_type='k3', entropy_weight=EW, kl_weight=KW)
    return out.loss


def a2c(d):
    return R.a2c_error_linear(R.a2c_linear_data(d['hidden'], d['lm_weight'], d['action'], d['value'], d['adv_tok'],
                                                d['return_'], d['weight']), value_weight=VW, entropy_weight=EW).loss


LOSSES = {'grpo': grpo, 'ppo': ppo, 'a2c': a2c}


def kernels(fn, d):
    """-> {kernel name (first 80 characters): launches} of one call"""
    clear(d)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    names = collections.Counter(e.name[:80] for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
                                and not e.name.startswith(('Memcpy', 'Memset')))
    return dict(sorted(names.items()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--repeats', type=int, default=30)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--losses', nargs='*', default=list(LOSSES))
    ap.add_argument('--workloads', nargs='*', default=[w[0] for w in WORKLOADS])
    args = ap.parse_args()
    print(json.dumps(card()), flush=True)
    R.ppo.LAZY_INFO = True
    for name, B, S, D, V, dtype in WORKLOADS:
        if name not in args.workloads:
            continue
        d = inputs(B, S, D, V, dtype, logits=False)
        for loss in args.losses:
            torch._dynamo.reset()
            compiled = torch.compile(LOSSES[loss], fullgraph=True)
            arms = {'eager': lambda f=LOSSES[loss]: f(d).backward(), 'compiled': lambda: compiled(d).backward()}
            for _ in range(args.warmup):
                for fn in arms.values():
                    clear(d)
                    fn()
            times = {a: [] for a in arms}
            for k in range(args.repeats):  # the order of the two arms flips from one repeat to the next
                for a in (list(arms) if k % 2 == 0 else list(arms)[::-1]):
                    times[a].append(event_ms(arms[a], d))
            diff = sorted(c - e for c, e in zip(times['compiled'], times['eager']))
            q = lambda f: round(diff[min(len(diff) - 1, int(f * len(diff)))], 3)
            print(json.dumps({'workload': name, 'loss': loss, 'compiled_minus_eager_ms': {
                'median': q(0.5), 'q25': q(0.25), 'q75': q(0.75), 'min': round(diff[0], 3), 'max': round(diff[-1], 3),
                'pairs': len(diff)}}), flush=True)
            for a, fn in arms.items():
                r = {'workload': name, 'loss': loss, 'arm': a, 'B': B, 'S': S, 'D': D, 'V': V, 'dtype': str(dtype)}
                r.update(summary(times[a]))
                r['peak_gb'] = peak_gb(fn, d)
                names = kernels(fn, d)
                r['kernels'] = sum(names.values())
                r['kernel_names'] = names
                print(json.dumps(r), flush=True)
        del d
        torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
