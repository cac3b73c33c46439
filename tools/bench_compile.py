"""What torch.compile buys a learner's loss step at minibatch sizes (the plugin-boundary operators, SAC's
``v_1step_td_error``, QR-DQN and continuous-action PPO), where the Python / ctypes path rather than the kernels
sets the time per call.  Each workload is one forward + backward loss step on CUDA tensors, timed as in
tools/host_overhead.py: wall-clock microseconds per call over a loop, device synchronised once per loop.  Three modes:
eager, ``torch.compile`` (default inductor) and ``torch.compile(mode="reduce-overhead")`` (the compiled step replayed as
a CUDA graph).  Also: the first (compiling) call's wall time, the CUDA kernels per call from ``torch.profiler`` in a
separate run, and for ``ppo_error`` at 320 rows the host entries that take the time per call (``torch.profiler``, CPU
activity, a third run).  The card's name and power limit are read in the same run.  ``ppo_error`` runs with ``LAZY_INFO`` (its two
monitors stay on the device) in every mode, so that no mode reads the device on the host.

    python tools/bench_compile.py > bench_compile.json
"""
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import di_engine_b200 as b2  # noqa: E402
from tests import cases  # noqa: E402

DEV = 'cuda:0'
api = b2.rl_utils


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [x.strip() for x in q.split(',')]
    except Exception:
        name, power = torch.cuda.get_device_name(0), 'unknown'
    return {'gpu': name, 'power_limit': power}


def wall(fn, n=300):
    for _ in range(20):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(n):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e6 / n


def kernels_per_call(fn, n=20):
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            fn()
        torch.cuda.synchronize()
    k = sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)
    return round(k / n, 2)


def host_breakdown(fn, n=50, top=10):
    """where a call's host time goes: the ``top`` host-side entries of ``torch.profiler`` (CPU activity, its own run) by
    self time, in µs per call, next to the profiled wall time per call (the profiler's own cost is in both)"""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU]) as prof:
        t0 = time.perf_counter()
        for _ in range(n):
            fn()
        torch.cuda.synchronize()
        wall_us = (time.perf_counter() - t0) * 1e6 / n
    rows = sorted(prof.key_averages(), key=lambda e: e.self_cpu_time_total, reverse=True)[:top]
    return {'profiled_wall_us': round(wall_us, 1),
            'top_self_us': [[e.key, round(e.self_cpu_time_total / n, 1), round(e.count / n, 2)] for e in rows]}


def to_dev(t):
    return {k: (v.to(DEV) if isinstance(v, torch.Tensor) else v) for k, v in t.items()}


def ppo_workload(rows):
    t = to_dev(cases.ppo_case(1, rows, 6)[1])
    ln = t['logit_new'].detach().requires_grad_(True)
    vn = t['value_new'].detach().requires_grad_(True)

    def loss(f):
        def step():
            ln.grad = vn.grad = None
            out, _ = f(api.ppo_data(ln, t['logit_old'], t['action'], vn, t['value_old'], t['adv'], t['return_'], None,
                                    None), 0.2)
            (out.policy_loss + 0.5 * out.value_loss - 0.01 * out.entropy_loss).backward()
        return step
    return api.ppo_error, loss


def qntd_workload():
    t = to_dev(cases.qntd_case(2, 64, 6, 3, done='bern')[1])
    q = t['q'].detach().requires_grad_(True)

    def loss(f):
        def step():
            q.grad = None
            out, _ = f(api.q_nstep_td_data(q, t['next_n_q'], t['action'], t['next_n_action'], t['reward'], t['done'], None),
                       0.99, 3)
            out.backward()
        return step
    return lambda *a: (lambda loss, per: (loss, per.detach()))(*api.q_nstep_td_error(*a)), loss


def vtrace_workload():
    t = to_dev(cases.vtrace_case(3, 64, 32, 6)[1])
    tgt = t['target_output'].detach().requires_grad_(True)
    v = t['value'].detach().requires_grad_(True)

    def loss(f):
        def step():
            tgt.grad = v.grad = None
            out = f(api.vtrace_data(tgt, t['behaviour_output'], t['action'], v, t['reward'], None))
            (out.policy_loss + 0.5 * out.value_loss - 0.01 * out.entropy_loss).backward()
        return step
    return api.vtrace_error_discrete_action, loss


def gae_workload():
    g = torch.Generator().manual_seed(3)
    T = 3200
    t = dict(value=torch.randn(T, generator=g), next_value=torch.randn(T, generator=g), reward=torch.randn(T, generator=g),
             done=(torch.rand(T, generator=g) < 0.003).float())
    t['traj_flag'] = t['done'].clone()
    t['traj_flag'][399::400] = 1.0
    t = to_dev(t)
    nv = t['next_value'].clone()

    def loss(f):
        def step():
            nv.copy_(t['next_value'])
            f(api.gae_data(t['value'], nv, t['reward'], t['done'], t['traj_flag']), 0.99, 0.95)
        return step
    return api.gae, loss


def v1td_workload():
    """SAC's critic loss at its batch of 256 (ding/policy/sac.py: one v_1step_td_error per Q head)"""
    g = torch.Generator().manual_seed(4)
    t = to_dev(dict(next_v=torch.randn(256, generator=g), reward=torch.randn(256, generator=g),
                    done=(torch.rand(256, generator=g) < 0.05).float()))
    v = torch.randn(256, generator=g).to(DEV).requires_grad_(True)

    def loss(f):
        def step():
            v.grad = None
            f(api.v_1step_td_data(v, t['next_v'], t['reward'], t['done'], None), 0.99)[0].backward()
        return step
    return lambda *a: (lambda loss, per: (loss, per.detach()))(*api.v_1step_td_error(*a)), loss


def qrdqn_workload():
    t = to_dev(cases.quantile_case(5, 'qrdqn', 64, 6, 32, 32, 3)[1])
    q = t['q'].detach().requires_grad_(True)

    def loss(f):
        def step():
            q.grad = None
            f(api.qrdqn_nstep_td_data(q, t['next_n_q'], t['action'], t['next_n_action'], t['reward'], t['done'], t['tau'],
                                      None), 0.99, 3)[0].backward()
        return step
    return lambda *a: (lambda loss, per: (loss, per.detach()))(*api.qrdqn_nstep_td_error(*a)), loss


def ppoc_workload():
    t = to_dev(cases.ppoc_case(6, 320, 6)[1])
    mu, sigma = (t[k].detach().requires_grad_(True) for k in ('mu_new', 'sigma_new'))
    vn = t['value_new'].detach().requires_grad_(True)

    def loss(f):
        def step():
            mu.grad = sigma.grad = vn.grad = None
            out, _ = f(api.ppo_data({'mu': mu, 'sigma': sigma}, {'mu': t['mu_old'], 'sigma': t['sigma_old']}, t['action'],
                                    vn, t['value_old'], t['adv'], t['return_'], None, None), 0.2)
            (out.policy_loss + 0.5 * out.value_loss - 0.01 * out.entropy_loss).backward()
        return step
    return api.ppo_error_continuous, loss


WORKLOADS = {
    'ppo_error_64x6': lambda: ppo_workload(64),
    'ppo_error_320x6': lambda: ppo_workload(320),
    'q_nstep_td_error_64x6_nstep3': qntd_workload,
    'vtrace_error_discrete_action_T64_B32': vtrace_workload,
    'gae_1d_n3200': gae_workload,
    'v_1step_td_error_256': v1td_workload,
    'qrdqn_nstep_td_error_64x6x32_nstep3': qrdqn_workload,
    'ppo_error_continuous_320x6': ppoc_workload,
}


BREAKDOWN = 'ppo_error_320x6'  # the workload whose host time is broken down by torch.profiler, in every mode


def main():
    api.ppo.LAZY_INFO = True
    res = card()
    res['torch'] = torch.__version__
    for name, make in WORKLOADS.items():
        fn, step_of = make()
        row = {}
        for mode, f in (('eager', fn), ('compile', torch.compile(fn, fullgraph=True)),
                        ('reduce_overhead', torch.compile(fn, fullgraph=True, mode='reduce-overhead'))):
            step = step_of(f)
            if mode != 'eager':
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                step()
                torch.cuda.synchronize()
                row[mode + '_first_call_s'] = round(time.perf_counter() - t0, 2)
            row[mode + '_us'] = round(wall(step), 1)
            row[mode + '_kernels_per_call'] = kernels_per_call(step)
            if name == BREAKDOWN:
                row[mode + '_host'] = host_breakdown(step)
        res[name] = row
        torch._dynamo.reset()
    print(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
