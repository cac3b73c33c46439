"""ScatterConnection (ding/torch_utils/network/scatter_connection.py:59-88), forward + backward of ``(out * out).mean()``
(the reference HPC test's loss, ding/hpc_rl/tests/test_scatter.py:54-57), on one GPU, two ways on the same CUDA tensors:

  reference   the reference module as it is (oracle/_ref, run on CUDA tensors: zero fill, repeat'ed int64 index, scatter_)
  library     di_engine_b200.ScatterConnection (csrc/scatter.cu)

Workloads (B, M, N, H, W, scatter_type):
  hpc_add / hpc_cover   the reference HPC test's shape (256, 256, 256, 16, 16): 256 entities into 256 cells, so the
                        backward stages g through shared memory (M * 8 >= H * W);
  football_add          gfootball_dqn_config's batch of 512, its spatial encoder's 22 players of 32 attributes into the
                        84 x 200 map (football_q_network.py:203,243): a 1.1 GB output and the backward's gather form;
  many_per_cell_add     1024 entities into 4 x 4 cells: 64 per cell, the sequential per-cell sums of the forward.

Per workload: device µs per call from CUDA events around a loop of ``--iters`` calls (median of ``--repeats`` loops, the
two implementations alternated); in a separate pass, the CUDA kernels per call and their summed time from torch.profiler,
and for the library the time of its own scatter kernels.  Their algorithmic bytes -- forward 4*B*M*N + 16*B*M read and
4*B*N*H*W written, backward 4*B*M*N gathered and 4*B*M*N written -- over that kernel time are set against a device copy of
the same traffic, timed the way tools/calib_copy.py times one.  The first JSON line names the card and its power limit.

    python tools/bench_scatter.py [--iters 50] [--warmup 5] [--repeats 5]
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
from oracle import ref_scatter  # noqa: E402

WORKLOADS = {
    'hpc_add': (256, 256, 256, 16, 16, 'add'),
    'hpc_cover': (256, 256, 256, 16, 16, 'cover'),
    'football_add': (512, 22, 32, 84, 200, 'add'),
    'many_per_cell_add': (64, 1024, 64, 4, 4, 'add'),
}


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i',
                        str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
    return {'device': torch.cuda.get_device_name(), 'nvidia_smi': q}


def inputs(B, M, N, H, W, seed=0):
    g = torch.Generator(device='cuda').manual_seed(seed)
    loc = torch.stack([torch.randint(0, H, (B, M), generator=g, device='cuda'),
                       torch.randint(0, W, (B, M), generator=g, device='cuda')], dim=2)
    return torch.randn(B, M, N, generator=g, device='cuda').requires_grad_(True), loc


def make_step(model, x, loc, H, W):

    def step():
        out = model(x, (H, W), loc)
        (out * out).mean().backward()
        x.grad = None

    return step


def device_us(step, iters):
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        step()
    t1.record()
    t1.synchronize()
    return t0.elapsed_time(t1) / iters * 1e3


def kernels(step, calls=5):
    """(CUDA kernels per call, their summed µs per call, summed µs per call of the library's scatter kernels)"""
    step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            step()
        torch.cuda.synchronize()
    ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and 'memcpy' not in e.name.lower()]
    own = [e for e in ev if 'b200rl' in e.name and 'scatter_' in e.name]
    return len(ev) / calls, sum(e.device_time for e in ev) / calls, sum(e.device_time for e in own) / calls


def algorithmic_bytes(B, M, N, H, W):
    return 4 * B * M * N + 16 * B * M + 4 * B * N * H * W + 8 * B * M * N


def copy_GBps(nbytes, iters=20):
    """a device copy of ``nbytes`` of traffic (half read, half written), as tools/calib_copy.py times one"""
    n = max(1, nbytes // 8)
    src, dst = torch.randn(n, device='cuda'), torch.empty(n, device='cuda')
    for _ in range(3):
        dst.copy_(src)
    us = statistics.median(device_us(lambda: dst.copy_(src), iters) for _ in range(3))
    return 8 * n / us / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--repeats', type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_scatter needs a GPU'
    print(json.dumps(card()), flush=True)
    with ref_scatter.network():
        Ref = ref_scatter.scatter_connection().ScatterConnection
        for name, (B, M, N, H, W, scatter_type) in WORKLOADS.items():
            x, loc = inputs(B, M, N, H, W)
            steps = {'reference': make_step(Ref(scatter_type), x, loc, H, W),
                     'library': make_step(b2.ScatterConnection(scatter_type), x, loc, H, W)}
            for s in steps.values():
                for _ in range(args.warmup):
                    s()
            res = {k: [] for k in steps}
            for _ in range(args.repeats):
                for k, s in steps.items():
                    res[k].append(device_us(s, args.iters))
            prof = {k: kernels(s) for k, s in steps.items()}
            for k in steps:
                row = {'workload': name, 'B_M_N_H_W': [B, M, N, H, W], 'scatter_type': scatter_type, 'impl': k,
                       'device_us': round(statistics.median(res[k]), 1),
                       'device_us_min_max': [round(min(res[k]), 1), round(max(res[k]), 1)],
                       'kernels_per_call': prof[k][0], 'kernel_us_per_call': round(prof[k][1], 1)}
                if k == 'library':
                    nbytes = algorithmic_bytes(B, M, N, H, W)
                    row['scatter_kernel_us_per_call'] = round(prof[k][2], 1)
                    row['algorithmic_bytes'] = nbytes
                    row['bytes_over_scatter_kernel_time_GBps'] = round(nbytes / prof[k][2] / 1e3, 1)
                    row['copy_of_same_traffic_GBps'] = round(copy_GBps(nbytes), 1)
                print(json.dumps(row), flush=True)
            del steps, x, loc
            torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
