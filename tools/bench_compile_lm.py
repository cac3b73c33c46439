"""What torch.compile costs the language-model losses at 16 x 1024 x 32768, where the kernels take milliseconds.

Under compile these losses recompute their gradient in the backward op instead of taking the forward-written one (see
INTEGRATION section 3d): the expected extra device time is one more read of logit_new, B * S * V * sizeof(T) bytes, at
the plain-copy read rate.  This script measures it.  Workloads, each one forward + backward, in fp32 and bf16:

    grpo      grpo_policy_error, loss.backward()
    rloo      rloo_policy_error (K = 4), loss.backward()
    ppo       ppo_policy_error with logit_pretrained: policy - 0.01 * entropy + 0.1 * kl
    a2c       a2c_error: policy + 0.5 * value - 0.01 * entropy
    logp      efficient_method, (lp * w).sum() backward

Modes: eager, ``torch.compile`` (inductor) and ``mode="reduce-overhead"``, all with ``LAZY_INFO`` (no host read of the
monitors).  Per workload and mode: device ms per forward + backward from CUDA events around 20 calls, the median of 5
repeats with the modes alternated in each repeat; the peak memory allocated by one call above its inputs; the CUDA kernels
per call from a separate ``torch.profiler`` run.  The card's name and power limit are read in the same run.

    python tools/bench_compile_lm.py > bench_compile_lm.json
"""
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import di_engine_b200 as b2  # noqa: E402

DEV = 'cuda:0'
api = b2.rl_utils
B, S, V = 16, 1024, 32768
CALLS, REPEATS = 20, 5


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [x.strip() for x in q.split(',')]
    except Exception:
        name, power = torch.cuda.get_device_name(0), 'unknown'
    return {'gpu': name, 'power_limit': power}


def inputs(kind, dtype):
    """(call(f) -> scalar to back-propagate, the leaves); every tensor made once, on the device"""
    g = torch.Generator(device=DEV).manual_seed(0)

    def randn(*shape, dt=torch.float32):
        return torch.randn(*shape, generator=g, device=DEV).to(dt)

    x = randn(B, S, V, dt=dtype).requires_grad_(True)
    act = torch.randint(0, V, (B, S), generator=g, device=DEV)
    w = (torch.rand(B, S, generator=g, device=DEV) > 0.1).float()
    if kind == 'grpo':
        data = api.grpo_policy_data(x, randn(B, S, V, dt=dtype), randn(B, S, V, dt=dtype), act, randn(B), w)
        return (lambda f: f['grpo'](data)[0]), [x]
    if kind == 'rloo':
        data = api.rloo_policy_data(x, randn(B, S, V, dt=dtype), act, randn(4, B // 4), w)
        return (lambda f: f['rloo'](data)[0]), [x]
    if kind == 'ppo':
        data = api.ppo_policy_data(x, randn(B, S, V, dt=dtype), act, randn(B, S), w, randn(B, S, V, dt=dtype))

        def ppo(f):
            loss = f['ppo'](data)[0]
            return loss.policy_loss - 0.01 * loss.entropy_loss + 0.1 * loss.kl_div

        return ppo, [x]
    if kind == 'a2c':
        v = randn(B, S).requires_grad_(True)
        data = api.a2c_data(x, act, v, randn(B, S), randn(B, S), w)

        def a2c(f):
            loss = f['a2c'](data)
            return loss.policy_loss + 0.5 * loss.value_loss - 0.01 * loss.entropy_loss

        return a2c, [x, v]
    return (lambda f: (f['logp'](x, act) * w).sum()), [x]


EAGER = {'grpo': api.grpo_policy_error, 'rloo': api.rloo_policy_error, 'ppo': api.ppo_policy_error, 'a2c': api.a2c_error,
         'logp': api.efficient_method}


def step(call, leaves, f):
    return torch.autograd.grad(call(f), leaves)


def device_ms(call, leaves, f):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(CALLS):
        step(call, leaves, f)
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / CALLS


def peak_bytes(call, leaves, f):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    grads = step(call, leaves, f)
    torch.cuda.synchronize()
    del grads
    return torch.cuda.max_memory_allocated() - base


def kernels_per_call(call, leaves, f, n=5):
    from torch.profiler import ProfilerActivity, profile
    step(call, leaves, f)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            step(call, leaves, f)
        torch.cuda.synchronize()
    k = sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)
    return round(k / n, 2)


def main():
    torch.cuda.init()
    info = card()
    api.ppo.LAZY_INFO = True
    torch._dynamo.config.cache_size_limit = 64
    modes = {'eager': EAGER,
             'compile': {k: torch.compile(f, fullgraph=True) for k, f in EAGER.items()},
             'reduce_overhead': {k: torch.compile(f, mode='reduce-overhead', fullgraph=True) for k, f in EAGER.items()}}
    rows = []
    for dtype in (torch.float32, torch.bfloat16):
        for kind in EAGER:
            call, leaves = inputs(kind, dtype)
            for fs in modes.values():  # compile, warm up, record the CUDA graph
                for _ in range(3):
                    step(call, leaves, fs)
            times = {m: [] for m in modes}
            for _ in range(REPEATS):
                for m, fs in modes.items():
                    times[m].append(device_ms(call, leaves, fs))
            row = {'workload': kind, 'dtype': str(dtype).split('.')[-1], 'shape': [B, S, V],
                   'logit_new_read_GB': B * S * V * x_size(dtype) / 1e9}
            for m, fs in modes.items():
                row[m] = {'device_ms': round(statistics.median(times[m]), 4),
                          'spread_ms': round(max(times[m]) - min(times[m]), 4),
                          'peak_MB': round(peak_bytes(call, leaves, fs) / 2 ** 20, 1),
                          'kernels_per_call': kernels_per_call(call, leaves, fs)}
            row['compile_over_eager'] = round(row['compile']['device_ms'] / row['eager']['device_ms'] - 1, 4)
            rows.append(row)
            print(json.dumps(dict(row, **info)), flush=True)
            del call, leaves
            torch.cuda.empty_cache()


def x_size(dtype):
    return torch.empty((), dtype=dtype).element_size()


if __name__ == '__main__':
    main()
