"""The layer-normalised LSTM (ding/torch_utils/network/rnn.py:131-239) on one GPU, two ways on the same CUDA tensors:

  reference   the reference module as it is (oracle/_ref): about 15 small kernels per step and layer
  library     the same module after ``install()``: the GEMMs on cuBLAS, one csrc/lstm.cu launch per step in each direction

Workloads, R2D2's Pong config (B = 64, hidden 512, burn-in 20, learn unroll 80; I = 512 stands for the encoder output):
  r2d2_unroll   the learner's per-step loop (q_learning.py:1031): 20 burn-in calls and 25 target-network burn-in calls
                under no_grad, 80 per-step calls with grad chained through list states and a backward through all 80, then
                80 target-network calls under no_grad;
  seq80         the same 80 steps as one seq_len = 80 call, forward + backward;
  collect       collector inference, T = 1, B = 8, no_grad.

Per workload and arm: device ms per workload from CUDA events around enough calls to last a second (median of
``--repeats`` loops, the arms alternated), host wall ms per workload from a host clock around the same loop ending in a
synchronise, and in a separate torch.profiler pass the CUDA kernels per workload.  Also the host ms per workload that the
reference's own ``_before_forward`` / ``_after_forward`` take (the list-state handling both arms keep), and, at the timed
sizes, the accuracy rule max|library - fp64| <= 2 max|reference - fp64| + 1e-6 max|fp64| for every output and gradient.
The first JSON line names the card and its power limit.

    python tools/bench_lstm.py [--repeats 5] [--out FILE]
"""
import argparse
import copy
import importlib
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
from oracle import ref_scatter  # noqa: E402

B, I, H = 64, 512, 512


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i',
                        str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
    return {'device': torch.cuda.get_device_name(), 'nvidia_smi': q}


def list_state(h, c):
    return [{'h': h[:, b:b + 1], 'c': c[:, b:b + 1]} for b in range(h.shape[1])]


def workloads(online, target, dt=torch.float32):
    g = torch.Generator(device='cuda').manual_seed(0)
    x = torch.randn(20 + 80, B, I, generator=g, device='cuda').to(dt)
    x8 = torch.randn(1, 8, I, generator=g, device='cuda').to(dt)
    h0, c0 = (torch.randn(1, B, H, generator=g, device='cuda').to(dt) * 0.5 for _ in range(2))

    def r2d2_unroll():
        with torch.no_grad():
            s = list_state(h0, c0)
            for t in range(20):
                _, s = online(x[t:t + 1], s)
            ts = list_state(h0, c0)
            for t in range(25):
                _, ts = target(x[t:t + 1], ts)
        online.zero_grad()
        ys = []
        for t in range(20, 100):
            y, s = online(x[t:t + 1], s)
            ys.append(y)
        y = torch.cat(ys)
        hT = torch.cat([d['h'] for d in s], 1)
        (y.square().mean() + hT.square().mean()).backward()
        with torch.no_grad():
            for t in range(20, 100):
                _, ts = target(x[t:t + 1], ts)
        return [y.detach(), hT.detach()] + [p.grad for p in online.parameters()]

    def seq80():
        online.zero_grad()
        y, s = online(x[20:], {'h': h0, 'c': c0}, list_next_state=False)
        (y.square().mean() + s['h'].square().mean()).backward()
        return [y.detach(), s['h'].detach(), s['c'].detach()] + [p.grad for p in online.parameters()]

    def collect():
        with torch.no_grad():
            y, s = online(x8, [None] * 8)
        return [y, torch.cat([d['h'] for d in s], 1)]

    return {'r2d2_unroll': r2d2_unroll, 'seq80': seq80, 'collect': collect}


def timed(fn, min_s=1.0):
    """(device ms, host wall ms) per call over enough calls to last min_s"""
    fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    n = max(3, int(min_s / max(time.perf_counter() - t0, 1e-6)))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    w0 = time.perf_counter()
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n, (time.perf_counter() - w0) * 1e3 / n


def kernels(fn):
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)


def rule(ours, ref32, ref64):
    worst = 0.0
    for a, r, d in zip(ours, ref32, ref64):
        a, r, d = a.double(), r.double(), d.double()
        bound = 2 * float((r - d).abs().max()) + 1e-6 * float(d.abs().max())
        err = float((a - d).abs().max())
        worst = max(worst, err / bound if bound > 0 else (0.0 if err == 0 else float('inf')))
    return worst  # <= 1 passes


def state_handling_ms(model, min_s=0.5):
    """host ms of the reference's _before_forward + _after_forward per call, at the per-step call's list state"""
    x = torch.zeros(1, B, I, device='cuda')
    h = torch.zeros(1, B, H, device='cuda')
    s = list_state(h, h)

    def one():
        st = model._before_forward(x, s)
        return model._after_forward(st, True)

    one()
    n, t0 = 0, time.perf_counter()
    while time.perf_counter() - t0 < min_s:
        one()
        n += 1
    return (time.perf_counter() - t0) * 1e3 / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--repeats', type=int, default=5)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    lines = [dict(card(), torch=torch.__version__)]
    print(json.dumps(lines[0]), flush=True)
    with ref_scatter.network():
        sys.modules['treetensor.torch'].Tensor = type('NoTreeTensor', (), {})
        rnn = importlib.import_module(ref_scatter.PACKAGE + '.rnn')
        torch.manual_seed(0)
        online = rnn.LSTM(I, H, 1, 'LN').cuda()
        target = copy.deepcopy(online)
        wl = workloads(online, target)
        per_call = {'r2d2_unroll': 20 + 25 + 80 + 80, 'seq80': 1, 'collect': 1}
        res = {k: {'reference': [], 'library': []} for k in wl}
        for _ in range(args.repeats):
            for arm in ('reference', 'library'):
                if arm == 'library':
                    b2.install()
                try:
                    for k, fn in wl.items():
                        res[k][arm].append(timed(fn))
                finally:
                    b2.uninstall()
        # accuracy at the timed sizes, and kernels per workload
        online64, target64 = copy.deepcopy(online).double(), copy.deepcopy(target).double()
        wl64 = workloads(online64, target64, torch.float64)
        for k, fn in wl.items():
            want = [t.clone() for t in wl64[k]()]
            ref32 = [t.clone() for t in fn()]
            k_ref = kernels(fn)
            b2.install()
            try:
                ours = [t.clone() for t in fn()]
                k_lib = kernels(fn)
            finally:
                b2.uninstall()
            line = {'workload': k, 'calls_per_workload': per_call[k], 'accuracy_rule_ratio': rule(ours, ref32, want)}
            for arm, kk in (('reference', k_ref), ('library', k_lib)):
                dev = statistics.median(r[0] for r in res[k][arm])
                wall = statistics.median(r[1] for r in res[k][arm])
                line[arm] = {'device_ms': round(dev, 4), 'host_wall_ms': round(wall, 4), 'kernels': kk,
                             'kernels_per_call': round(kk / per_call[k], 2)}
            lines.append(line)
            print(json.dumps(line), flush=True)
        sh = state_handling_ms(online)
        line = {'state_handling_ms_per_call': round(sh, 4),
                'r2d2_unroll_state_handling_ms': round(sh * per_call['r2d2_unroll'], 3)}
        lines.append(line)
        print(json.dumps(line), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write('\n'.join(json.dumps(l) for l in lines) + '\n')


if __name__ == '__main__':
    main()
