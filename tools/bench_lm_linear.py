"""grpo_policy_error_linear and token_logp_linear (rl_utils/lm_linear.py) against the logit-tensor forms they replace, on
one GPU.  Three arms, alternated within each repeat on the same card:

  linear     grpo_policy_error_linear (chunked GEMMs + csrc/vocab.cu in place)
  logits     F.linear + the library's grpo_policy_error (the whole (B, S, V) logits and their gradient)
  reference  F.linear + the reference's grpo_policy_error with efficient_method (oracle/ref_lm.py; skipped where it does
             not fit in memory or the reference is not available)

Workloads: 16 x 1024 tokens, D = 3584, V = 152 064 bf16 (Qwen2-7B's lm_head); D = 4096, V = 32 768 in bf16 and fp32.
Per arm and workload: forward + backward of GRPO (beta = 0.1) with gradients to hidden and lm_weight, and the log-prob
call under no_grad (the rollout / reference-model form: token_logp_linear, or F.linear + efficient_method).  Printed as
JSON lines after one line naming the card and its power limit:

  ms          device time from CUDA events around one call, median (min, max) of --repeats
  peak_gb     torch.cuda.max_memory_allocated during the call, above what was allocated before it (inputs, parameters)
  gemm_ms / row_ms / other_ms   the device-time split from a separate torch.profiler run of one call
  gemm_tflops 3 * 2 * N * D * V flops (logits, dH, dW) over gemm_ms
  row_gbs     the row kernel's floor, 2 * V * sizeof(T) bytes per token, over its time

--budgets MiB [MiB ...] times the linear arm alone at each chunk budget (ops.LM_CHUNK_BYTES) instead.

    python tools/bench_lm_linear.py [--repeats 5] [--warmup 1] [--budgets 128 256 512 1024]
"""
import argparse
import json
import os
import statistics
import sys

import torch
import torch.nn.functional as F
from torch.profiler import ProfilerActivity, profile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import di_engine_b200 as b2  # noqa: E402
from di_engine_b200 import ops  # noqa: E402
from oracle import ref_lm  # noqa: E402
from tools.bench_soft_td import card  # noqa: E402

R = b2.rl_utils
WORKLOADS = [('qwen2_7b_bf16', 16, 1024, 3584, 152064, torch.bfloat16),
             ('d4096_v32768_bf16', 16, 1024, 4096, 32768, torch.bfloat16),
             ('d4096_v32768_fp32', 16, 1024, 4096, 32768, torch.float32)]


def inputs(B, S, D, V, dtype, logits):
    g = torch.Generator(device='cuda').manual_seed(0)
    h = torch.randn(B, S, D, device='cuda', generator=g, dtype=dtype).requires_grad_(True)
    w = (torch.randn(V, D, device='cuda', generator=g) / D ** 0.5).to(dtype).requires_grad_(True)
    d = {'hidden': h, 'lm_weight': w, 'action': torch.randint(0, V, (B, S), device='cuda', generator=g),
         'adv': torch.randn(B, device='cuda', generator=g),
         'weight': (torch.rand(B, S, device='cuda', generator=g) > 0.1).float()}
    with torch.no_grad():
        for k, s in (('old', 0.05), ('ref', 0.1)):
            hk = (h.float() + s * torch.randn(B, S, D, device='cuda', generator=g)).to(dtype)
            d['logp_' + k] = R.token_logp_linear(hk, w, d['action'])
            if logits:
                d['logit_' + k] = F.linear(hk, w)
    return d


def arm_step(arm, d, ref):
    def linear():
        loss, _ = R.grpo_policy_error_linear(R.grpo_linear_data(d['hidden'], d['lm_weight'], d['logp_old'], d['logp_ref'],
                                                                d['action'], d['adv'], d['weight']), beta=0.1)
        loss.backward()

    def logits():
        z = F.linear(d['hidden'], d['lm_weight'])
        loss, _ = R.grpo_policy_error(R.grpo_policy_data(z, d['logit_old'], d['logit_ref'], d['action'], d['adv'],
                                                         d['weight']), beta=0.1)
        loss.backward()

    def reference():
        z = F.linear(d['hidden'], d['lm_weight'])
        m = ref['grpo']
        loss, _ = m.grpo_policy_error(m.grpo_policy_data(z, d['logit_old'], d['logit_ref'], d['action'], d['adv'],
                                                         d['weight']), ref['log_prob_utils'].efficient_method, beta=0.1)
        loss.backward()

    def logp_linear():
        with torch.no_grad():
            R.token_logp_linear(d['hidden'], d['lm_weight'], d['action'])

    def logp_logits():
        with torch.no_grad():
            R.efficient_method(F.linear(d['hidden'], d['lm_weight']), d['action'])

    def logp_reference():
        with torch.no_grad():
            ref['log_prob_utils'].efficient_method(F.linear(d['hidden'], d['lm_weight']), d['action'])

    return {'linear': (linear, logp_linear), 'logits': (logits, logp_logits),
            'reference': (reference, logp_reference)}[arm]


def clear(d):
    d['hidden'].grad = None
    d['lm_weight'].grad = None


def event_ms(fn, d):
    clear(d)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def peak_gb(fn, d):
    clear(d)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return round((torch.cuda.max_memory_allocated() - base) / 1e9, 3)


def split(fn, d):
    """device ms of GEMMs, of the library's row kernels and of everything else in one call"""
    clear(d)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    t = {'gemm': 0.0, 'row': 0.0, 'other': 0.0}
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        n = e.name.lower()
        us = e.time_range.elapsed_us()
        if 'vocab_rows_kernel' in n:
            t['row'] += us
        elif any(k in n for k in ('gemm', 'nvjet', 'cutlass', 'xmma', 'sm90_', 'cublas')):
            t['gemm'] += us
        else:
            t['other'] += us
    return {k: round(v / 1e3, 3) for k, v in t.items()}


def summary(ms):
    return {'ms': round(statistics.median(ms), 3), 'min': round(min(ms), 3), 'max': round(max(ms), 3)}


def run_workload(name, B, S, D, V, dtype, arms, ref, repeats, warmup):
    N, T = B * S, torch.tensor([], dtype=dtype).element_size()
    d = inputs(B, S, D, V, dtype, logits=arms != ['linear'])
    steps = {a: arm_step(a, d, ref) for a in arms}
    live = {}
    for a in arms:  # a call that runs out of memory drops its arm (the reference at Qwen's vocabulary, say)
        try:
            for _ in range(warmup):
                for fn in steps[a]:
                    clear(d)
                    fn()
            torch.cuda.synchronize()
            live[a] = steps[a]
        except torch.cuda.OutOfMemoryError:
            clear(d)
            torch.cuda.empty_cache()
            print(json.dumps({'workload': name, 'arm': a, 'skipped': 'out of memory'}), flush=True)
    times = {(a, k): [] for a in live for k in (0, 1)}
    for _ in range(repeats):
        for a in live:
            for k in (0, 1):
                times[(a, k)].append(event_ms(live[a][k], d))
    rows = []
    for a in live:
        for k, what in ((0, 'grpo_fwd_bwd'), (1, 'logp_no_grad')):
            r = {'workload': name, 'arm': a, 'call': what, 'B': B, 'S': S, 'D': D, 'V': V, 'dtype': str(dtype)}
            r.update(summary(times[(a, k)]))
            r['peak_gb'] = peak_gb(live[a][k], d)
            sp = split(live[a][k], d)
            r.update({'gemm_ms': sp['gemm'], 'row_ms': sp['row'], 'other_ms': sp['other']})
            gemms = 3 if k == 0 else 1
            if sp['gemm'] > 0:
                r['gemm_tflops'] = round(gemms * 2 * N * D * V / (sp['gemm'] * 1e-3) / 1e12, 1)
            if a != 'reference' and sp['row'] > 0:
                floor = N * (2 if k == 0 else 1) * V * T  # the log-prob pass reads the logits only
                r['row_gbs'] = round(floor / (sp['row'] * 1e-3) / 1e9, 1)
            rows.append(r)
            print(json.dumps(r), flush=True)
    del d, steps, live
    torch.cuda.empty_cache()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--repeats', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=1)
    ap.add_argument('--budgets', type=int, nargs='*', help='MiB: time the linear arm at each chunk budget')
    ap.add_argument('--workloads', nargs='*', default=[w[0] for w in WORKLOADS])
    args = ap.parse_args()
    print(json.dumps(card()), flush=True)
    ref = None
    if not args.budgets and ref_lm.available():
        ctx = ref_lm.modules()
        ref = ctx.__enter__()
    for name, B, S, D, V, dtype in WORKLOADS:
        if name not in args.workloads:
            continue
        if args.budgets:
            for mib in args.budgets:
                ops.LM_CHUNK_BYTES = mib << 20
                for r in run_workload(name, B, S, D, V, dtype, ['linear'], None, args.repeats, args.warmup):
                    print(json.dumps({'budget_mib': mib, 'call': r['call'], 'ms': r['ms'], 'peak_gb': r['peak_gb']}),
                          flush=True)
            continue
        arms = ['linear', 'logits'] + (['reference'] if ref is not None else [])
        run_workload(name, B, S, D, V, dtype, arms, ref, args.repeats, args.warmup)


if __name__ == '__main__':
    main()
