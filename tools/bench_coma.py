"""COMAPolicy's loss (``coma_error``, ding/rl_utils/coma.py:10-58), forward + backward of
0.001 * policy + q_value_loss - 0.01 * entropy (policy/coma.py:213-214), on one GPU, three ways on the same CUDA tensors:

  reference           the reference function as it is (oracle/_ref, run on CUDA tensors)
  reference+install   the same function after ``install()``: its lambda-return already runs on the library's scan
  library             di_engine_b200's ``coma_error``

Shapes (T, B, A, N): the SMAC configs' (10, 32, 10, 18), (20, 32, 8, 14) and (20, 32, 2, 70), the reference test's
(128, 4, 8, 32), and one large (128, 256, 8, 32).  logit and q_value are leaves that require grad and target_q_value does
not, as in COMAPolicy (policy/coma.py:206-207); logits carry COMAPolicy's -9999999 action mask.

Per shape and implementation: wall µs per call over a loop of ``--iters`` calls (>= 300) with one device synchronise at
its end, and device µs per call from CUDA events around the same kind of loop (median of ``--repeats`` loops;
reference+install and library alternated, the reference after ``uninstall()``); in a separate pass, CUDA kernels per call and their summed time counted by torch.profiler (the
whole step: the mask assignment and the loss weighting included) and, for the library, the time of its own COMA kernels,
and for the large shape the algorithmic bytes over that kernel time against 3.35 TB/s.  The
first JSON line names the card and its power limit.

    python tools/bench_coma.py [--iters 300] [--warmup 30] [--repeats 5]
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
from oracle import ref_coma  # noqa: E402

SHAPES = {'smac_3s5z': (10, 32, 10, 18), 'smac_mmm': (20, 32, 8, 14), 'smac_2c64zg': (20, 32, 2, 70),
          'reference_test': (128, 4, 8, 32), 'large': (128, 256, 8, 32)}
HBM_BPS = 3.35e12  # H100 SXM data sheet


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i',
                        str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
    return {'device': torch.cuda.get_device_name(), 'nvidia_smi': q}


def inputs(T, B, A, N, seed=0):
    g = torch.Generator(device='cuda').manual_seed(seed)
    action = torch.randint(0, N, (T, B, A), generator=g, device='cuda')
    legal = torch.rand(T, B, A, N, generator=g, device='cuda') < 0.7
    legal.scatter_(-1, action.unsqueeze(-1), True)
    return {'logit_raw': torch.randn(T, B, A, N, generator=g, device='cuda'), 'legal': legal, 'action': action,
            'q_value': torch.randn(T, B, A, N, generator=g, device='cuda').requires_grad_(True),
            'target_q_value': torch.randn(T, B, A, N, generator=g, device='cuda'),
            'reward': torch.rand(T, B, generator=g, device='cuda'), 'weight': None}


def make_step(coma_data, coma_error, x):
    leaf = x['logit_raw'].clone().requires_grad_(True)
    mask = ~x['legal']

    def step():
        logit = leaf * 1.0  # a non-leaf, so the mask assignment is legal, as for the actor's output
        logit[mask] = -9999999
        loss = coma_error(coma_data(logit, x['action'], x['q_value'], x['target_q_value'], x['reward'], x['weight']),
                          0.99, 0.8)
        (0.001 * loss.policy_loss + 1 * loss.q_value_loss - 0.01 * loss.entropy_loss).backward()
        leaf.grad = None
        x['q_value'].grad = None

    return step


def wall_us(step, iters):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(iters):
        step()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / iters * 1e6


def device_us(step, iters):
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        step()
    t1.record()
    t1.synchronize()
    return t0.elapsed_time(t1) / iters * 1e3


def kernels(step, calls=10):
    """(CUDA kernels per call, their summed µs per call, summed µs per call of the library's COMA kernels)"""
    step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            step()
        torch.cuda.synchronize()
    ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and 'memcpy' not in e.name.lower()
          and 'memset' not in e.name.lower()]
    own = [e for e in ev if 'coma' in e.name]
    return len(ev) / calls, sum(e.device_time for e in ev) / calls, sum(e.device_time for e in own) / calls


def algorithmic_bytes(T, B, A, N):
    """forward + backward of the library: logit and q_value read once and d logit / d q_value written once (T*B*A*N floats
    each), the gathered target column, action (twice), reward, adv and dq per row"""
    R, cells = T * B * A, T * B * A * N
    return 4 * cells * 4 + R * (4 + 8 * 2 + 4 * 3) + T * B * 4


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=300)
    ap.add_argument('--warmup', type=int, default=30)
    ap.add_argument('--repeats', type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_coma needs a GPU'
    assert args.iters >= 300
    print(json.dumps(card()), flush=True)
    with ref_coma.module() as ref:
        ref_fn = ref.coma_error  # the function object; install() rebinds the lambda-return in its module's globals
        for name, (T, B, A, N) in SHAPES.items():
            x = inputs(T, B, A, N)
            steps = {'reference': make_step(ref.coma_data, ref_fn, x)}
            b2.install()
            try:
                steps['reference+install'] = make_step(ref.coma_data, ref_fn, x)
                steps['library'] = make_step(b2.coma_data, b2.coma_error, x)
                order = ['reference+install', 'library']
                for s in order:
                    for _ in range(args.warmup):
                        steps[s]()
                res = {k: {'wall': [], 'device': []} for k in steps}
                for _ in range(args.repeats):
                    for k in order:
                        res[k]['wall'].append(wall_us(steps[k], args.iters))
                        res[k]['device'].append(device_us(steps[k], args.iters))
                prof = {k: kernels(steps[k]) for k in order}
            finally:
                b2.uninstall()
            for _ in range(args.warmup):
                steps['reference']()
            for _ in range(args.repeats):
                res['reference']['wall'].append(wall_us(steps['reference'], args.iters))
                res['reference']['device'].append(device_us(steps['reference'], args.iters))
            prof['reference'] = kernels(steps['reference'])
            for k in steps:
                row = {'shape': name, 'T_B_A_N': [T, B, A, N], 'impl': k,
                       'wall_us': round(statistics.median(res[k]['wall']), 1),
                       'device_us': round(statistics.median(res[k]['device']), 1),
                       'device_us_min_max': [round(min(res[k]['device']), 1), round(max(res[k]['device']), 1)],
                       'kernels_per_call': prof[k][0], 'kernel_us_per_call': round(prof[k][1], 1)}
                if k == 'library':
                    row['coma_kernel_us_per_call'] = round(prof[k][2], 1)
                if k == 'library' and name == 'large':
                    nbytes = algorithmic_bytes(T, B, A, N)
                    row['algorithmic_bytes'] = nbytes
                    row['bytes_over_coma_kernel_time_TBps'] = round(nbytes / (prof[k][2] * 1e-6) / 1e12, 3)
                    row['share_of_3.35TBps'] = round(nbytes / (prof[k][2] * 1e-6) / HBM_BPS, 3)
                print(json.dumps(row), flush=True)


if __name__ == '__main__':
    main()
