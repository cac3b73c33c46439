"""The TD losses of the entropy-regularised value learners, forward + backward, on one GPU: the reference functions
(oracle/_ref, run on CUDA tensors) against di_engine_b200, at the shipped sizes.

  M-DQN   m_q_1step_td_error     B = 32,  N = 6 (Atari)
  SQL     q_nstep_sql_td_error   B = 64,  N = 2 (CartPole) and N = 4 (LunarLander), nstep 1
  SAC     q_v_1step_td_error     B = 256, N = 6, twin critic (two calls, two backward passes, as policy/sac.py:262-278)

Each timing is a host clock around K iterations that end in a device synchronise, after W warm-up iterations; the median
and spread over R such runs are printed as JSON lines, after one line naming the card and its power limit.  A separate,
untimed pass per case counts the kernel launches of one iteration with torch.profiler.

    python tools/bench_soft_td.py [--iters 500] [--warmup 50] [--repeats 7]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

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
        t0 = time.perf_counter()
        for _ in range(iters):
            step()
        torch.cuda.synchronize()
        runs.append((time.perf_counter() - t0) / iters * 1e6)
    return {'median_us': round(statistics.median(runs), 2), 'min_us': round(min(runs), 2), 'max_us': round(max(runs), 2)}


def launches(step):
    """kernel launches and memcpy / memset operations of one iteration (after a warm-up call)"""
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


def mdqn_step(api, B, N, seed):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(B, N, generator=g).cuda().requires_grad_(True)
    tqc, tqn = torch.randn(B, N, generator=g).cuda(), torch.randn(B, N, generator=g).cuda()
    act = torch.randint(0, N, (B, ), generator=g).cuda()
    reward, done = torch.randn(B, generator=g).cuda(), torch.randint(0, 2, (B, ), generator=g).float().cuda()
    weight = torch.rand(B, generator=g).cuda()

    def step():
        q.grad = None
        loss, _, _, _ = api.m_q_1step_td_error(api.m_q_1step_td_data(q, tqc, tqn, act, reward, done, weight), 0.99, 0.03,
                                               0.9)
        loss.backward()
    return step


def sql_step(api, B, N, seed):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(B, N, generator=g).cuda().requires_grad_(True)
    nq = torch.randn(B, N, generator=g).cuda()
    act, nact = torch.randint(0, N, (B, ), generator=g).cuda(), torch.randint(0, N, (B, ), generator=g).cuda()
    reward, done = torch.rand(1, B, generator=g).cuda(), torch.randint(0, 2, (B, ), generator=g).float().cuda()

    def step():
        q.grad = None
        loss, _, rec = api.q_nstep_sql_td_error(api.q_nstep_td_data(q, nq, act, nact, reward, done, None), 0.99, 0.12,
                                                nstep=1)
        rec.mean()  # policy/sql.py:148
        loss.backward()
    return step


def sac_step(api, B, N, seed):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(2, B, N, generator=g).cuda().requires_grad_(True)
    v = torch.randn(B, generator=g).cuda()
    act = torch.randint(0, N, (B, ), generator=g).cuda()
    reward, done = torch.randn(B, generator=g).cuda(), torch.randint(0, 2, (B, ), generator=g).float().cuda()

    def step():
        q.grad = None
        l0, e0 = api.q_v_1step_td_error(api.q_v_1step_td_data(q[0], v, act, reward, done, None), 0.99)
        l1, e1 = api.q_v_1step_td_error(api.q_v_1step_td_data(q[1], v, act, reward, done, None), 0.99)
        (e0 + e1) / 2  # the twin critic's priority, policy/sac.py:274
        l0.backward()
        l1.backward()
    return step


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=500)
    ap.add_argument('--warmup', type=int, default=50)
    ap.add_argument('--repeats', type=int, default=7)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_soft_td: needs a CUDA device")
    ref = ref_loader.load()
    print(json.dumps(card()))
    cases = [('m_q_1step_td_error B=32 N=6', mdqn_step, 32, 6),
             ('q_nstep_sql_td_error B=64 N=2 nstep=1', sql_step, 64, 2),
             ('q_nstep_sql_td_error B=64 N=4 nstep=1', sql_step, 64, 4),
             ('q_v_1step_td_error x2 (twin critic) B=256 N=6', sac_step, 256, 6)]
    for name, make, B, N in cases:
        for impl, api in (('reference', ref), ('b200', b2.rl_utils)):
            step = make(api, B, N, 0)
            res = timed(step, args.iters, args.warmup, args.repeats)
            print(json.dumps(dict(case=name, impl=impl, **res, **launches(step))))


if __name__ == '__main__':
    main()
