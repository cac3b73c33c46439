"""PPOFPolicy's advantage recompute (ding/policy/ppof.py:160-210) on one GPU: the reference's lines (the reference functions
from oracle/_ref, run on CUDA tensors) against ``ppof_gae_returns``, on the same tensors, for each value_norm mode at

  n = 128, 400   one sequence of n_sample steps (the shipped PPOF configs)
  n = 3200       8 environments x 400 steps in one sequence
  (T, B) = (128, 4096)

The critic's output is taken as given, so the time is the recompute alone: decode, gae, returns, encode and, in 'baseline',
the copy of the returns to the host that RunningMeanStd.update reads (:208; ``ppof_gae_returns`` hands back three device
floats instead).  Each timing is CUDA events around K calls after W warm-up calls; the median and spread over R such runs are
printed as JSON lines, after one line naming the card and its power limit.  A separate, untimed pass counts each path's
kernel launches and copies per call with torch.profiler.

    python tools/bench_ppof.py [--iters 50] [--ref-iters 5] [--warmup 3] [--repeats 5]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import di_engine_b200 as b2  # noqa: E402
from oracle import ref_loader  # noqa: E402

MODES = ('baseline', 'value_rescale', 'symlog', 'popart')
SHAPES = [(128, ), (400, ), (3200, ), (128, 4096)]
GAMMA, LAMBDA, STD = 0.99, 0.95, np.float64(1.7320508)


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


def reference_lines(ref, mode, pred, next_pred, reward, done, traj_flag, mu, sigma):
    """ppof.py:171-210 as the policy runs them (the model call replaced by its outputs)"""
    value, next_value = pred, next_pred
    if mode == 'popart':
        reward = (reward - mu) / sigma
    elif mode == 'value_rescale':
        value, next_value = ref.value_inv_transform(value), ref.value_inv_transform(next_value)
    elif mode == 'symlog':
        value, next_value = ref.inv_symlog(value), ref.inv_symlog(next_value)
    else:
        value, next_value = value * STD, next_value * STD
    adv = ref.gae(ref.gae_data(value, next_value, reward, done, traj_flag), GAMMA, LAMBDA)
    ret = value + adv
    if mode == 'value_rescale':
        value, ret = ref.value_transform(value), ref.value_transform(ret)
    elif mode == 'symlog':
        value, ret = ref.symlog(value), ref.symlog(ret)
    elif mode == 'baseline':
        value /= STD
        ret /= STD
        ret.cpu().numpy()  # what RunningMeanStd.update receives
    return adv, value, ret


def make(shape, mode, seed=0):
    g = torch.Generator(device='cuda').manual_seed(seed)
    scale = 3.0 if mode in ('symlog', 'value_rescale') else 1.0
    t = {
        'pred': torch.randn(*shape, generator=g, device='cuda') * scale,
        'next_pred': torch.randn(*shape, generator=g, device='cuda') * scale,
        'reward': torch.randn(*shape, generator=g, device='cuda'),
        'done': (torch.rand(*shape, generator=g, device='cuda') < 0.01).float(),
        'mu': torch.randn(1, generator=g, device='cuda'),
        'sigma': torch.rand(1, generator=g, device='cuda') + 0.5,
    }
    t['traj_flag'] = t['done'].clone()
    t['traj_flag'][-1] = 1.0
    if mode == 'popart' and len(shape) == 1:
        t['pred'], t['next_pred'] = t['pred'][:, None], t['next_pred'][:, None]  # PopArt's (n, 1) prediction
    return t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=50)
    ap.add_argument('--ref-iters', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--repeats', type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_ppof.py needs a CUDA device')
    ref = ref_loader.load()
    print(json.dumps(card()))
    for shape in SHAPES:
        for mode in MODES:
            t = make(shape, mode)

            def ours():
                return b2.ppof_gae_returns(b2.gae_data(t['pred'], t['next_pred'], t['reward'], t['done'], t['traj_flag']),
                                           GAMMA, LAMBDA, mode, std=STD if mode == 'baseline' else None,
                                           popart_mu=t['mu'], popart_sigma=t['sigma'])

            def theirs():
                return reference_lines(ref, mode, t['pred'], t['next_pred'], t['reward'], t['done'], t['traj_flag'],
                                       t['mu'], t['sigma'])

            a, b = ours(), theirs()
            agree = bool(torch.equal(a.adv, b[0]))
            row = {'mode': mode, 'shape': list(shape), 'adv_bit_identical': agree}
            row['ours'] = dict(timed(ours, args.iters, args.warmup, args.repeats), **launches(ours))
            row['reference'] = dict(timed(theirs, args.ref_iters, 1, args.repeats), **launches(theirs))
            row['speedup'] = round(row['reference']['median_us'] / row['ours']['median_us'], 1)
            print(json.dumps(row), flush=True)


if __name__ == '__main__':
    main()
