"""grpo_policy_error_linear, token_logp_linear, ppo_policy_error_linear and a2c_error_linear (rl_utils/lm_linear.py)
against the logit-tensor forms they replace, on one GPU.  Three arms, alternated within each repeat on the same card:

  linear     the hidden-state loss (chunked GEMMs + csrc/vocab.cu in place)
  logits     F.linear + the library's logit-form loss (the whole (B, S, V) logits and their gradient; PPO also holds
             logit_old and logit_pretrained)
  reference  F.linear + the reference's loss (GRPO with efficient_method: oracle/ref_lm.py; PPO / A2C:
             oracle/ref_loader.py; skipped where it does not fit in memory or the reference is not available)

Workloads: 16 x 1024 tokens, D = 3584, V = 152 064 bf16 (Qwen2-7B's lm_head); D = 4096, V = 32 768 in bf16 and fp32.
Per arm and workload, forward + backward with gradients to hidden and lm_weight (and A2C's value) of:

  --loss grpo  GRPO (beta = 0.1), and the log-prob call under no_grad (the rollout / reference-model form:
               token_logp_linear, or F.linear + efficient_method)
  --loss ppo   ppo_policy_error, clip 0.2, k3 KL with kl_weight 0.1, entropy_weight 0.01; and the same without the
               entropy term (entropy_bonus=False)
  --loss a2c   a2c_error, value_weight 0.5, entropy_weight 0.01

Printed as JSON lines after one line naming the card and its power limit:

  ms          device time from CUDA events around one call, median (min, max) of --repeats
  peak_gb     torch.cuda.max_memory_allocated during the call, above what was allocated before it (inputs, parameters)
  gemm_ms / row_ms / other_ms   the device-time split from a separate torch.profiler run of one call
  gemm_tflops 3 * 2 * N * D * V flops (logits, dH, dW) over gemm_ms
  row_gbs     the row kernel's floor, 2 * V * sizeof(T) bytes per token, over its time

--budgets MiB [MiB ...] times the linear arm alone at each chunk budget (ops.LM_CHUNK_BYTES) instead.

    python tools/bench_lm_linear.py [--loss grpo] [--repeats 5] [--warmup 1] [--budgets 128 256 512 1024]
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
from oracle import ref_loader, ref_lm  # noqa: E402
from tools.bench_soft_td import card  # noqa: E402

R = b2.rl_utils
WORKLOADS = [('qwen2_7b_bf16', 16, 1024, 3584, 152064, torch.bfloat16),
             ('d4096_v32768_bf16', 16, 1024, 4096, 32768, torch.bfloat16),
             ('d4096_v32768_fp32', 16, 1024, 4096, 32768, torch.float32)]


EW, KW, VW = 0.01, 0.1, 0.5  # entropy_weight, kl_weight (k3), value_weight


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
    # PPO / A2C: per-token advantage, the reference policy as the pretrained one, a value head's output and returns
    d['adv_tok'] = torch.randn(B, S, device='cuda', generator=g)
    d['value'] = torch.randn(B, S, device='cuda', generator=g).requires_grad_(True)
    d['return_'] = torch.randn(B, S, device='cuda', generator=g)
    return d


def grpo_calls(d, ref):
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

    return {'linear': [('grpo_fwd_bwd', linear, 3, 2), ('logp_no_grad', logp_linear, 1, 1)],
            'logits': [('grpo_fwd_bwd', logits, 3, 2), ('logp_no_grad', logp_logits, 1, 1)],
            'reference': [('grpo_fwd_bwd', reference, 3, 2), ('logp_no_grad', logp_reference, 1, 1)]}


def ppo_calls(d, ref):
    def linear(ent):
        def fn():
            loss, _ = R.ppo_policy_error_linear(
                R.ppo_policy_linear_data(d['hidden'], d['lm_weight'], d['logp_old'], d['action'], d['adv_tok'],
                                         d['weight'], d['logp_ref']), entropy_bonus=ent, kl_type='k3',
                entropy_weight=EW if ent else 0.0, kl_weight=KW)
            loss.loss.backward()
        return fn

    def logits(m, ent):
        def fn():
            z = F.linear(d['hidden'], d['lm_weight'])
            p, _ = m.ppo_policy_error(m.ppo_policy_data(z, d['logit_old'], d['action'], d['adv_tok'], d['weight'],
                                                        d['logit_ref']), entropy_bonus=ent, kl_type='k3')
            (p.policy_loss - (EW if ent else 0.0) * p.entropy_loss + KW * p.kl_div).backward()
        return fn

    out = {'linear': [('ppo_fwd_bwd', linear(True), 3, 2), ('ppo_noent_fwd_bwd', linear(False), 3, 2)],
           'logits': [('ppo_fwd_bwd', logits(R, True), 3, 2), ('ppo_noent_fwd_bwd', logits(R, False), 3, 2)]}
    if ref is not None:
        out['reference'] = [('ppo_fwd_bwd', logits(ref, True), 3, 2), ('ppo_noent_fwd_bwd', logits(ref, False), 3, 2)]
    return out


def a2c_calls(d, ref):
    def linear():
        loss = R.a2c_error_linear(R.a2c_linear_data(d['hidden'], d['lm_weight'], d['action'], d['value'], d['adv_tok'],
                                                    d['return_'], d['weight']), value_weight=VW, entropy_weight=EW)
        loss.loss.backward()

    def logits(m):
        def fn():
            z = F.linear(d['hidden'], d['lm_weight'])
            a = m.a2c_error(m.a2c_data(z, d['action'], d['value'], d['adv_tok'], d['return_'], d['weight']))
            (a.policy_loss + VW * a.value_loss - EW * a.entropy_loss).backward()
        return fn

    out = {'linear': [('a2c_fwd_bwd', linear, 3, 2)], 'logits': [('a2c_fwd_bwd', logits(R), 3, 2)]}
    if ref is not None:
        out['reference'] = [('a2c_fwd_bwd', logits(ref), 3, 2)]
    return out


def clear(d):
    d['hidden'].grad = None
    d['lm_weight'].grad = None
    d['value'].grad = None


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


def run_workload(name, B, S, D, V, dtype, arms, calls, ref, repeats, warmup):
    """calls(d, ref) -> {arm: [(call name, fn, GEMMs per call, passes of the row floor)]}"""
    N, T = B * S, torch.tensor([], dtype=dtype).element_size()
    d = inputs(B, S, D, V, dtype, logits=arms != ['linear'])
    table = calls(d, ref)
    steps = {a: table[a] for a in arms if a in table}
    live = {}
    for a in steps:  # a call that runs out of memory drops its arm (the reference at Qwen's vocabulary, say)
        try:
            for _ in range(warmup):
                for _, fn, _, _ in steps[a]:
                    clear(d)
                    fn()
            torch.cuda.synchronize()
            live[a] = steps[a]
        except torch.cuda.OutOfMemoryError:
            clear(d)
            torch.cuda.empty_cache()
            print(json.dumps({'workload': name, 'arm': a, 'skipped': 'out of memory'}), flush=True)
    times = {(a, k): [] for a in live for k in range(len(live[a]))}
    for _ in range(repeats):
        for a in live:
            for k, (_, fn, _, _) in enumerate(live[a]):
                times[(a, k)].append(event_ms(fn, d))
    rows = []
    for a in live:
        for k, (what, fn, gemms, passes) in enumerate(live[a]):
            r = {'workload': name, 'arm': a, 'call': what, 'B': B, 'S': S, 'D': D, 'V': V, 'dtype': str(dtype)}
            r.update(summary(times[(a, k)]))
            r['peak_gb'] = peak_gb(fn, d)
            sp = split(fn, d)
            r.update({'gemm_ms': sp['gemm'], 'row_ms': sp['row'], 'other_ms': sp['other']})
            if sp['gemm'] > 0:
                r['gemm_tflops'] = round(gemms * 2 * N * D * V / (sp['gemm'] * 1e-3) / 1e12, 1)
            if a != 'reference' and sp['row'] > 0:
                floor = N * passes * V * T  # the log-prob pass reads the logits only
                r['row_gbs'] = round(floor / (sp['row'] * 1e-3) / 1e9, 1)
            rows.append(r)
            print(json.dumps(r), flush=True)
    del d, steps, live, table
    torch.cuda.empty_cache()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--loss', choices=['grpo', 'ppo', 'a2c'], default='grpo')
    ap.add_argument('--repeats', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=1)
    ap.add_argument('--budgets', type=int, nargs='*', help='MiB: time the linear arm at each chunk budget')
    ap.add_argument('--workloads', nargs='*', default=[w[0] for w in WORKLOADS])
    args = ap.parse_args()
    print(json.dumps(card()), flush=True)
    calls = {'grpo': grpo_calls, 'ppo': ppo_calls, 'a2c': a2c_calls}[args.loss]
    ref = None
    if not args.budgets and args.loss == 'grpo' and ref_lm.available():
        ctx = ref_lm.modules()
        ref = ctx.__enter__()
    elif not args.budgets and args.loss != 'grpo' and ref_loader.available():
        ref = ref_loader.load()
    for name, B, S, D, V, dtype in WORKLOADS:
        if name not in args.workloads:
            continue
        if args.budgets:
            for mib in args.budgets:
                ops.LM_CHUNK_BYTES = mib << 20
                for r in run_workload(name, B, S, D, V, dtype, ['linear'], calls, None, args.repeats, args.warmup):
                    print(json.dumps({'budget_mib': mib, 'call': r['call'], 'ms': r['ms'], 'peak_gb': r['peak_gb']}),
                          flush=True)
            continue
        arms = ['linear', 'logits'] + (['reference'] if ref is not None else [])
        run_workload(name, B, S, D, V, dtype, arms, calls, ref, args.repeats, args.warmup)


if __name__ == '__main__':
    main()
