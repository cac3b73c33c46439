"""DQfD / R2D3 loss, forward + backward, on one GPU: the reference functions (oracle/_ref, run on CUDA tensors) against
di_engine_b200.

  (a) one dqfd_nstep_td_error call, B = 32, N = 6, nstep = 3 (the DQfD Atari configs);
  (b) R2D3's 35-step loop (r2d3.py:322-388), B = 64, N = 6, nstep = 5, value rescale on: the reference loop, the drop-in
      called per step, and dqfd_nstep_td_error_sequence.

Each timing is a host clock around K iterations that end in a device synchronise, after W warm-up iterations; the
median and spread over R such runs are printed as JSON lines, after one line naming the card and its power limit.

    python tools/bench_dqfd.py [--iters 200] [--warmup 20] [--repeats 7]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import di_engine_b200 as b2  # noqa: E402
from oracle import ref_loader  # noqa: E402

FIELDS = ('q', 'next_n_q', 'action', 'next_n_action', 'reward', 'done', 'done_one_step', 'weight', 'new_n_q_one_step',
          'next_n_action_one_step', 'is_expert')


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i',
                        str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
    return {'device': torch.cuda.get_device_name(), 'nvidia_smi': q}


def inputs(lead, N, nstep, seed):
    g = torch.Generator().manual_seed(seed)
    t = {
        'q': torch.randn(*lead, N, generator=g),
        'next_n_q': torch.randn(*lead, N, generator=g),
        'action': torch.randint(0, N, lead, generator=g),
        'next_n_action': torch.randint(0, N, lead, generator=g),
        'reward': torch.rand(*((nstep, ) + lead if len(lead) == 1 else (lead[0], nstep, lead[1])), generator=g),
        'done': torch.randint(0, 2, lead, generator=g).float(),
        'done_one_step': torch.randint(0, 2, lead, generator=g).float(),
        'weight': torch.rand(*lead, generator=g),
        'new_n_q_one_step': torch.randn(*lead, N, generator=g),
        'next_n_action_one_step': torch.randint(0, N, lead, generator=g),
        'is_expert': torch.randint(0, 2, lead, generator=g).float(),
    }
    return {k: v.cuda() for k, v in t.items()}


def timed(step, iters, warmup, repeats):
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    runs = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        for _ in range(iters):
            step()
        torch.cuda.synchronize()
        runs.append((time.perf_counter() - t0) / iters * 1e6)
    return {'median_us': round(statistics.median(runs), 2), 'min_us': round(min(runs), 2), 'max_us': round(max(runs), 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=200)
    ap.add_argument('--warmup', type=int, default=20)
    ap.add_argument('--repeats', type=int, default=7)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_dqfd: needs a CUDA device")
    ref = ref_loader.load()
    print(json.dumps(card()))
    K, W, R = args.iters, args.warmup, args.repeats

    # (a) one DQfD call
    t = inputs((32, ), 6, 3, 0)
    q = t['q'].clone().requires_grad_(True)

    def one(api):
        def step():
            q.grad = None
            data = api.dqfd_nstep_td_data(q, *[t[k] for k in FIELDS[1:]])
            loss, _, _ = api.dqfd_nstep_td_error(data, 0.99, 1.0, 1.0, 0.8, nstep=3)
            loss.backward()
        return step

    for impl, api in (('reference', ref), ('b200', b2.rl_utils)):
        print(json.dumps(dict(case='dqfd_nstep_td_error B=32 N=6 nstep=3', impl=impl, **timed(one(api), K, W, R))))

    # (b) R2D3's loop, value rescale on
    T, B, N, nstep, gamma = 35, 64, 6, 5, 0.997
    s = inputs((T, B), N, nstep, 1)
    vg = torch.rand(T, B, generator=torch.Generator().manual_seed(2)).cuda() * 0.1 + 0.9
    qs = s['q'].clone().requires_grad_(True)
    lambda1, lambda2, margin, lambda_one = 1.0, 1.0, 0.8, 1.0

    def loop(api):
        def step():
            qs.grad = None
            loss, td_error = [], []
            for i in range(T):
                d = api.dqfd_nstep_td_data(qs[i], *[s[k][i] for k in FIELDS[1:]])
                l, e, _ = api.dqfd_nstep_td_error_with_rescale(d, gamma, lambda1, lambda2, margin, lambda_one, nstep,
                                                               False, value_gamma=vg[i])
                loss.append(l)
                td_error.append(e)
            loss = sum(loss) / (len(loss) + 1e-8)
            torch.max(torch.stack(td_error), dim=0)  # the priority's reductions (r2d3.py:386-388)
            torch.sum(torch.stack(td_error), dim=0)
            loss.backward()
        return step

    def seq():
        qs.grad = None
        data = b2.dqfd_nstep_td_seq_data(qs, *[s[k] for k in FIELDS[1:]])
        loss, _, _, _ = b2.dqfd_nstep_td_error_sequence(data, gamma, lambda1, lambda2, lambda_one, margin, nstep,
                                                        value_gamma=vg, rescale=True)
        loss.backward()

    name = 'R2D3 loop T=35 B=64 N=6 nstep=5 rescale'
    for impl, step in (('reference loop', loop(ref)), ('b200 per-step loop', loop(b2.rl_utils)),
                       ('b200 sequence form', seq)):
        print(json.dumps(dict(case=name, impl=impl, **timed(step, max(K // 10, 5), max(W // 4, 3), R))))


if __name__ == '__main__':
    main()
