"""What torch.compile buys the value-based losses that now trace as custom ops (DQfD, R2D2's sequence loop, M-DQN, soft
Q-learning, discrete SAC's critic and FQF's fraction loss), at the minibatch sizes of the shipped configs, where the
Python / ctypes path rather than the kernels sets the time per call.  Each workload is one forward + backward loss step on
CUDA tensors, the per-sample errors, priorities and statistics leaving detached as a learner takes them.  Measured as
tools/bench_compile.py measures: wall-clock microseconds per call over a loop, device synchronised once per loop, in
eager mode, under ``torch.compile`` (default inductor) and under ``mode="reduce-overhead"``; the first (compiling) call's
wall time; the CUDA kernels per call from ``torch.profiler`` in a separate run.  The card's name and power limit are read
in the same run.

    python tools/bench_compile_td.py > bench_compile_td.json
"""
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torch  # noqa: E402

import di_engine_b200 as b2  # noqa: E402
from bench_compile import card, kernels_per_call, wall  # noqa: E402

DEV = 'cuda:0'
api = b2.rl_utils


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _dev(*ts):
    return [t.to(DEV) for t in ts]


def dqfd_workload(B=64, N=6, nstep=3):
    """DQfDPolicy's minibatch (dizoo/atari dqfd configs: batch 64, nstep 3)"""
    g = _g(1)
    q = torch.randn(B, N, generator=g).to(DEV).requires_grad_(True)
    nq, nq1 = _dev(torch.randn(B, N, generator=g), torch.randn(B, N, generator=g))
    act, nact, nact1 = _dev(*(torch.randint(0, N, (B, ), generator=g) for _ in range(3)))
    reward, = _dev(torch.randn(nstep, B, generator=g))
    done, expert = _dev((torch.rand(B, generator=g) < 0.05).float(), (torch.rand(B, generator=g) < 0.5).float())

    def fn(data):
        loss, td, stats = api.dqfd_nstep_td_error(data, 0.99, 1.0, 1.0, 0.8, nstep=nstep)
        return loss, td.detach(), torch.stack(stats).detach()

    def step_of(f):
        def step():
            q.grad = None
            f(api.dqfd_nstep_td_data(q, nq, act, nact, reward, done, done, None, nq1, nact1, expert))[0].backward()
        return step
    return fn, step_of


def r2d2_workload(T=80, B=64, N=6, nstep=5):
    """R2D2's (T, B) unroll in one call (dizoo/atari r2d2 configs: unroll 80, batch 64, nstep 5, value rescaling)"""
    g = _g(2)
    q = torch.randn(T, B, N, generator=g).to(DEV).requires_grad_(True)
    nq, = _dev(torch.randn(T, B, N, generator=g))
    act, nact = _dev(torch.randint(0, N, (T, B), generator=g), torch.randint(0, N, (T, B), generator=g))
    reward, done, weight = _dev(torch.randn(T, nstep, B, generator=g), (torch.rand(T, B, generator=g) < 0.01).float(),
                                torch.rand(T, B, generator=g))

    def fn(data):
        loss, prio, td = api.q_nstep_td_error_sequence(data, 0.997, nstep=nstep, rescale=True)
        return loss, prio, td.detach()

    def step_of(f):
        def step():
            q.grad = None
            f(api.q_nstep_td_seq_data(q, nq, act, nact, reward, done, weight))[0].backward()
        return step
    return fn, step_of


def soft_workload(kind, B, N=6, nstep=1):
    """M-DQN (batch 32), SQL and discrete SAC's critic (batch 64) on a six-action head"""
    g = _g(3)
    q = torch.randn(B, N, generator=g).to(DEV).requires_grad_(True)
    tq, nq = _dev(torch.randn(B, N, generator=g), torch.randn(B, N, generator=g))
    act, nact = _dev(torch.randint(0, N, (B, ), generator=g), torch.randint(0, N, (B, ), generator=g))
    reward, done, v = _dev(torch.randn(nstep, B, generator=g), (torch.rand(B, generator=g) < 0.05).float(),
                           torch.randn(B, generator=g))

    def fn(data):
        if kind == 'mdqn':
            loss, td, gap, clip = api.m_q_1step_td_error(data, 0.99, 0.03, 0.9)
            return loss, td.detach(), gap, clip
        if kind == 'sql':
            loss, td, rec = api.q_nstep_sql_td_error(data, 0.99, 0.1, nstep=nstep)
            return loss, td.detach(), rec
        loss, td = api.q_v_1step_td_error(data, 0.99)
        return loss, td.detach()

    def data():
        if kind == 'mdqn':
            return api.m_q_1step_td_data(q, tq, nq, act, reward[0], done, None)
        if kind == 'sql':
            return api.q_nstep_td_data(q, nq, act, nact, reward, done, None)
        return api.q_v_1step_td_data(q, v, act, reward[0], done, None)

    def step_of(f):
        def step():
            q.grad = None
            f(data())[0].backward()
        return step
    return fn, step_of


def fraction_workload(B=32, N=32, A=6):
    """FQFPolicy's fraction loss (dizoo/atari fqf configs: batch 32, 32 quantiles)"""
    g = _g(4)
    q_tau_i, = _dev(torch.randn(B, N - 1, A, generator=g))
    q_value = torch.randn(B, N, A, generator=g).to(DEV).requires_grad_(True)
    p = torch.softmax(torch.randn(B, N, generator=g), 1)
    quantiles = torch.cat([torch.zeros(B, 1), p.cumsum(1)], 1).to(DEV).requires_grad_(True)
    act, = _dev(torch.randint(0, A, (B, ), generator=g))

    def step_of(f):
        def step():
            quantiles.grad = None
            f(q_tau_i, q_value, quantiles, act).backward()
        return step
    return api.fqf_calculate_fraction_loss, step_of


WORKLOADS = {
    'dqfd_nstep_td_error_64x6_nstep3': dqfd_workload,
    'q_nstep_td_error_sequence_T80_B64x6_nstep5_rescale': r2d2_workload,
    'm_q_1step_td_error_32x6': lambda: soft_workload('mdqn', 32),
    'm_q_1step_td_error_64x6': lambda: soft_workload('mdqn', 64),
    'q_nstep_sql_td_error_64x6': lambda: soft_workload('sql', 64),
    'q_v_1step_td_error_64x6': lambda: soft_workload('qv', 64),
    'fqf_calculate_fraction_loss_32x32x6': fraction_workload,
}


def main():
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
        res[name] = row
        torch._dynamo.reset()
    print(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
