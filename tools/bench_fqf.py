"""FQFPolicy's loss block (ding/policy/fqf.py:239-248), forward + both backward passes, on one GPU: the reference functions
(oracle/_ref, run on CUDA tensors) against di_engine_b200 (``fqf_calculate_fraction_loss`` and ``fqf_nstep_td_error``), on the
same tensors, at the shipped sizes and one large batch.

  Pong      B = 32,    N = 32 quantiles, A = 6 actions (dizoo/atari/config/serial/pong/pong_fqf_config.py)
  CartPole  B = 64,    N = 32, A = 2
  large     B = 65536, N = 32, A = 6

The block takes the model's outputs as given (leaf tensors standing for q, quantiles and q_tau_i, plus a softmax-cumsum of a
learnable tensor for the quantiles as the head builds them), so the time is the loss work alone.  Each timing is CUDA events
around K blocks after W warm-up blocks; the median and spread over R such runs are printed as JSON lines, after one line
naming the card and its power limit.  A separate, untimed pass per case counts the kernel launches of one block with
torch.profiler, and for the fraction loss alone.

    python tools/bench_fqf.py [--iters 200] [--warmup 30] [--repeats 7]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
from torch.profiler import ProfilerActivity, profile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import di_engine_b200 as b2  # noqa: E402
from oracle import ref_loader  # noqa: E402


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i',
                        str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
    return {'device': torch.cuda.get_device_name(), 'nvidia_smi': q}


def timed(step, iters, warmup, repeats):
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    runs = []
    for _ in range(repeats):
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(iters):
            step()
        t1.record()
        t1.synchronize()
        runs.append(t0.elapsed_time(t1) / iters * 1e3)
    return {'median_us': round(statistics.median(runs), 2), 'min_us': round(min(runs), 2), 'max_us': round(max(runs), 2)}


def launches(step):
    """kernel launches and memcpy / memset operations of one call (after a warm-up call)"""
    step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    kernels = copies = 0
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        name = e.name.lower()
        if 'memcpy' in name or 'memset' in name:
            copies += 1
        else:
            kernels += 1
    return {'kernels': kernels, 'memcpy_memset': copies}


def make(B, N, A, seed=0):
    g = torch.Generator(device='cuda').manual_seed(seed)
    return {
        'frac': torch.randn(B, N, generator=g, device='cuda').requires_grad_(True),
        'q': torch.randn(B, N, A, generator=g, device='cuda').requires_grad_(True),
        'q_tau_i': torch.randn(B, N - 1, A, generator=g, device='cuda'),
        'target_q': torch.randn(B, N, A, generator=g, device='cuda'),
        'action': torch.randint(0, A, (B, ), generator=g, device='cuda'),
        'target_action': torch.randint(0, A, (B, ), generator=g, device='cuda'),
        'reward': torch.randn(1, B, generator=g, device='cuda'),
        'done': torch.randint(0, 2, (B, ), generator=g, device='cuda').float(),
        'weight': torch.rand(B, generator=g, device='cuda'),
    }


def block_step(api, t, fraction_only=False):
    def step():
        t['frac'].grad = None
        t['q'].grad = None
        p = torch.softmax(t['frac'], 1)
        quantiles = torch.cat([torch.zeros_like(p[:, :1]), torch.cumsum(p, 1)], 1)
        hats = (quantiles[:, 1:] + quantiles[:, :-1]).detach() / 2.
        fraction_loss = api.fqf_calculate_fraction_loss(t['q_tau_i'], t['q'], quantiles, t['action'])
        if fraction_only:
            fraction_loss.backward()
            return
        data_n = api.fqf_nstep_td_data(t['q'], t['target_q'], t['action'], t['target_action'], t['reward'], t['done'],
                                       hats, t['weight'])
        quantile_loss, _ = api.fqf_nstep_td_error(data_n, 0.99, nstep=1, kappa=1.0)
        fraction_loss.backward(retain_graph=True)
        quantile_loss.backward()
    return step


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=200)
    ap.add_argument('--warmup', type=int, default=30)
    ap.add_argument('--repeats', type=int, default=7)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fqf: needs a CUDA device")
    ref = ref_loader.load()
    print(json.dumps(card()))
    for name, B, N, A in (('pong', 32, 32, 6), ('cartpole', 64, 32, 2), ('large', 65536, 32, 6)):
        t = make(B, N, A)
        for impl, api in (('reference', ref), ('b200', b2.rl_utils)):
            res = timed(block_step(api, t), args.iters, args.warmup, args.repeats)
            frac = timed(block_step(api, t, True), args.iters, args.warmup, args.repeats)
            print(json.dumps(dict(case=name, B=B, N=N, A=A, impl=impl, block=dict(**res, **launches(block_step(api, t))),
                                  fraction_only=dict(**frac, **launches(block_step(api, t, True))))))


if __name__ == '__main__':
    main()
