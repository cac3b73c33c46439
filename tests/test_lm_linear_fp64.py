"""The hidden-state losses of rl_utils/lm_linear.py (grpo / rloo_policy_error_linear, ppo_policy_error_linear in all four
flag combinations, a2c_error_linear, token_logp_linear) against a float64 reference, on the token rows of
tests/test_vocab_fp64.py and at every hand-off of ``ops.lm_chunks_``.

An exact factorisation makes the kernel's in-place d loss / d logits visible.  With H = I (N x N, as (B, S, N)) and
W = Z^T (V x N) for a logit tensor Z drawn by ``test_vocab_fp64.gen_rows``, F.linear(H, W) is Z bit for bit in fp32 and in
bf16 (each output is 1 * z plus exact zeros; TF32 is switched off here, as is cuBLAS's reduced-precision bf16
reduction, whose partial sums would not be fp32), and dW = dZ^T H is dZ^T bit for bit: the returned dW *is* the kernel's
gradient buffer, checked element by element and row by row with ``test_vocab_fp64.compare_regimes``.  A gradient element
that the kernel fails to overwrite keeps a stale logit.  dH = dZ W is a real GEMM, checked as a tensor.  Where N is too
large for D = N, H row n is e_(n mod P) (P = 512; fp32 only): logits repeat every P rows, while actions, weights and
log-probabilities are per token, and dW (a sum of N / P gradient rows) is checked as a tensor.  Every case first checks
the identity on the device.  The masked regime uses -1e30 / -1e4, never -inf (-inf * 0 is NaN inside a GEMM).

Per-token log-probabilities (logp_old, logp_ref, logp_pretrained) are the fp32 values the call receives, and the
references take those same values upcast (``grpo_oracle.run64`` / ``ppo_lm_oracle.run64``'s ``lp_*`` arguments).  On-policy
rows take logp_old from ``token_logp_linear`` on the same hidden states, as the first step of a GRPO / PPO iteration does;
an all-on-policy case must give clipfrac 0 exactly.  A2C's reference is ``oracle/rl_oracle.a2c_error``.

Rule: ``compare64`` / ``compare_regimes`` with K = 8 against the float32 restatement, per regime, for the scalars, per-token
lp, dZ (read through dW) and d value.  dH and the periodic dW: the same bound against the fp32 GEMM of the float32
reference's dZ (bf16: the same bf16 GEMM, unchunked, of the kernel's own dZ, itself checked element by element, since bf16
operands round dZ by far more than an fp32 GEMM does).  Upstream gradients g = 1,
nextafter(1, 2), 0.37, -2, 0: dX(g) must equal (dX(1).float() * g).to(dtype) bit for bit (for fp32 and nextafter(1, 2) that
differs from dX(1) in every non-zero entry, so a skipped scale shows), with hidden, lm_weight and both requiring grad;
a repeated backward (the recompute path) gives 2 * dX(g) bit for bit; the same plan repeats bit for bit, another plan
stays within the bound; the forward under no_grad (no row cache, no gradient buffer) gives the same scalars.  Each case
prints its worst ratio per regime.

The cases straddle every hand-off: V at the row plan's edges (fp32 1, 3, 1027, 56 320, 56 324, 152 063 -- the row cache's
edge and the in-place re-read of the uncached part; bf16 1, 7, 1003, 112 640, 112 648, 152 064), one chunk, many 128-row
chunks, chunks with more rows than any grid (a CTA loops), a last chunk shorter than the grid (idle CTAs store zero
partials), the largest plan ``ops.lm_chunk_plan`` accepts for PPO's five sums, S = 1, S = 127..129 (sequences across
chunk boundaries), S = 1500 (more than 10 chunks, more than lm_seq_kernel's 256 threads), B above lm_seq_kernel's grid,
weights none / 0-1 / fractional, a zero-weight sequence in separate cases (NaN loss and NaN rows as float64's), RLOO with
K = 2, 3, 64 and B.  The CPU part checks those claims from the chunk plan at 132 SMs, the identity in fp32, and that the
comparison rejects one corrupted dZ element, one row left as stale logits and two rows swapped across a chunk boundary.

Dense hidden states at D = 1, 63 and 4096 (fp32 and bf16), a strided ``hidden`` and a transposed ``lm_weight`` run
under test_lm_linear's composition rule."""
import contextlib
import functools
import math
from collections import OrderedDict

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from di_engine_b200 import ops
from oracle import rl_oracle
from tests import grpo_oracle as go
from tests import ppo_lm_oracle as po
from tests import test_vocab_fp64 as vf
from tests.test_offpolicy_fp64 import K, compare64, policy_terms

assert K == 8.0  # the bound of the fp64 suites, shared, not loosened here
DEV = 'cuda'
F32, BF16 = torch.float32, torch.bfloat16
P_PERIOD = 512
SMS = 132  # the H100 SXM's SM count, for the CPU's plan claims
LM_SEQ_PER_SM = 2048 // 256  # lm_seq_kernel: 256 threads, at most 2048 resident per SM
EW, KW, VW = 0.01, 0.1, 0.5  # entropy_weight, kl_weight, value_weight
MASKS = (-1e30, -1e4)
NO_OLD = ('plain', 'shift', 'peaked', 'flat', 'masked', 'large')  # the regimes without an old policy (A2C, log p)


# ----------------------------------------------------------------------------------------------------------------
# the case table
# ----------------------------------------------------------------------------------------------------------------
def _c(kind, dtype, B, S, V, w=None, K=0, rows=None, periodic=False, ent=False, kl=None, dc=None, names=None, zero=False,
       claims=()):
    return dict(kind=kind, dtype=dtype, B=B, S=S, V=V, w=w, K=K, rows=rows, periodic=periodic, ent=ent, kl=kl, dc=dc,
                names=names, zero=zero, claims=set(claims))


def _ppo_grid():
    out = OrderedDict()
    i = 0
    for ent, kl in ((False, None), (True, None), (False, 'k1'), (False, 'k2'), (False, 'k3'), (True, 'k1'), (True, 'k2'),
                    (True, 'k3')):
        for dc in (None, 2.0):
            dtype, V = ((F32, 1027), (BF16, 1003))[i % 2]
            rows = 128 if i % 4 < 2 else None
            name = 'ppo_%s_v%d_%s_%s_%s%s' % ('f32' if dtype == F32 else 'bf16', V, 'ent' if ent else 'noent',
                                              kl or 'nokl', 'dc' if dc else 'nodc', '_c128' if rows else '')
            out[name] = _c('ppo', dtype, 23, 23, V, (None, 'mask', 'frac')[i % 3], rows=rows, ent=ent, kl=kl, dc=dc,
                           claims=('many', 'straddle', 'short_last') if rows else ('one', ))
            i += 1
    return out


PPO_LIMIT_CHUNKS = ops._WS_PARTIAL_WORDS // (128 * 5)  # 128-row chunks of PPO's five sums: 399 fit, 400 do not

CASES = OrderedDict([
    # GRPO
    ('grpo_f32_v1_one', _c('grpo', F32, 16, 8, 1, 'frac', claims=('one', ))),
    ('grpo_f32_v3_s129_c128', _c('grpo', F32, 5, 129, 3, rows=128, claims=('many', 'straddle', 'short_last'))),
    ('grpo_f32_v1027_s1500_c128', _c('grpo', F32, 2, 1500, 1027, 'frac', rows=128,
                                     claims=('many', 'straddle', 'short_last', 'long_seq'))),
    ('grpo_f32_v56320_r131', _c('grpo', F32, 131, 1, 56320, 'frac', claims=('one', ))),
    ('grpo_f32_v56324_s127_c128', _c('grpo', F32, 2, 127, 56324, 'mask', rows=128, claims=('straddle', 'short_last'))),
    ('grpo_f32_v152063_r3', _c('grpo', F32, 1, 3, 152063, 'frac', claims=('one', ))),
    ('grpo_f32_v2048_c128_zero_seq', _c('grpo', F32, 7, 19, 2048, 'mask', rows=128, zero=True,
                                        claims=('straddle', 'short_last'))),
    ('grpo_bf16_v1_r1', _c('grpo', BF16, 1, 1, 1, claims=('one', ))),
    ('grpo_bf16_v7_b1104_c1024', _c('grpo', BF16, 1104, 2, 7, 'frac', rows=1024, claims=('loop', 'b_grid'))),
    ('grpo_bf16_v1003_s1500_c128', _c('grpo', BF16, 2, 1500, 1003, 'frac', rows=128,
                                      claims=('many', 'straddle', 'short_last', 'long_seq'))),
    ('grpo_bf16_v112640_r131', _c('grpo', BF16, 131, 1, 112640, 'frac', claims=('one', ))),
    ('grpo_bf16_v112648_s129_c128', _c('grpo', BF16, 2, 129, 112648, rows=128, claims=('many', 'straddle', 'short_last'))),
    ('grpo_bf16_v152064_r3', _c('grpo', BF16, 3, 1, 152064, claims=('one', ))),
    ('grpo_f32_v3_zero_seq', _c('grpo', F32, 5, 30, 3, 'mask', zero=True, claims=('one', ))),
    ('grpo_bf16_v1003_onpolicy_c128', _c('grpo', BF16, 4, 40, 1003, 'frac', rows=128, names=('onpolicy', ),
                                         claims=('straddle', 'short_last'))),
    # RLOO
    ('rloo_f32_k2_v1027_s133_c128', _c('rloo', F32, 4, 133, 1027, 'frac', K=2, rows=128,
                                       claims=('many', 'straddle', 'short_last'))),
    ('rloo_f32_k3_v4100', _c('rloo', F32, 6, 22, 4100, 'mask', K=3, claims=('one', ))),
    ('rloo_f32_k2_v1027_zero_seq', _c('rloo', F32, 6, 10, 1027, 'mask', K=2, zero=True, claims=('one', ))),
    ('rloo_bf16_k64_v9_c128', _c('rloo', BF16, 192, 4, 9, K=64, rows=128, claims=('many', ))),
    ('rloo_bf16_kB_v8200_s9', _c('rloo', BF16, 8, 9, 8200, 'frac', K=8, claims=('one', ))),
    # PPO: the four flag combinations x dual clip x k1 / k2 / k3, then the edges
    *_ppo_grid().items(),
    ('ppo_f32_v3_s1_c128_ent_k1_dc', _c('ppo', F32, 300, 1, 3, 'frac', rows=128, ent=True, kl='k1', dc=2.0,
                                        claims=('many', 'short_last'))),
    ('ppo_f32_v56324_s127_c128_ent_k3_dc', _c('ppo', F32, 2, 127, 56324, 'frac', rows=128, ent=True, kl='k3', dc=2.0,
                                              claims=('straddle', 'short_last'))),
    ('ppo_f32_v152063_r3_ent_k2', _c('ppo', F32, 1, 3, 152063, 'mask', ent=True, kl='k2', claims=('one', ))),
    ('ppo_f32_v1027_onpolicy_ent_k3', _c('ppo', F32, 7, 19, 1027, 'frac', ent=True, kl='k3', names=('onpolicy', ),
                                         claims=('one', ))),
    ('ppo_bf16_v112648_s129_c128_ent_k1_dc', _c('ppo', BF16, 2, 129, 112648, None, rows=128, ent=True, kl='k1', dc=2.0,
                                                claims=('many', 'straddle', 'short_last'))),
    ('ppo_bf16_v152064_r3_noent_k3', _c('ppo', BF16, 3, 1, 152064, 'frac', kl='k3', claims=('one', ))),
    # its 512 logit rows repeat 100 times, so one row's rounding counts 100 times in each sum: kl_far's e^20 k3 terms would
    # let a few rows' logsumexp ulps decide the scalars' bound (the exact cases cover kl_far)
    ('ppo_f32_v1027_limit_ent_k3_dc', _c('ppo', F32, 32, PPO_LIMIT_CHUNKS * 4, 1027, 'frac', rows=128, periodic=True,
                                         ent=True, kl='k3', dc=2.0, names=vf.REGIMES[:-1],
                                         claims=('many', 'straddle', 'long_seq', 'limit'))),
    # A2C
    ('a2c_f32_v1_one', _c('a2c', F32, 16, 8, 1, 'frac', claims=('one', ))),
    ('a2c_f32_v1027_s1500_c128', _c('a2c', F32, 2, 1500, 1027, 'mask', rows=128,
                                    claims=('many', 'straddle', 'short_last', 'long_seq'))),
    ('a2c_f32_v56320_r131', _c('a2c', F32, 131, 1, 56320, 'frac', claims=('one', ))),
    ('a2c_f32_v56324_s127_c128', _c('a2c', F32, 2, 127, 56324, None, rows=128, claims=('straddle', 'short_last'))),
    ('a2c_f32_v152063_r3', _c('a2c', F32, 1, 3, 152063, 'frac', claims=('one', ))),
    ('a2c_bf16_v7_b1104_c1024', _c('a2c', BF16, 1104, 2, 7, 'mask', rows=1024, claims=('loop', ))),
    ('a2c_bf16_v112640_r131', _c('a2c', BF16, 131, 1, 112640, None, claims=('one', ))),
    ('a2c_bf16_v112648_s129_c128', _c('a2c', BF16, 2, 129, 112648, 'frac', rows=128,
                                      claims=('many', 'straddle', 'short_last'))),
    ('a2c_bf16_v152064_r3', _c('a2c', BF16, 3, 1, 152064, 'frac', claims=('one', ))),
    # the log-prob forward / backward
    ('logp_f32_v3_s129_c128', _c('logp', F32, 5, 129, 3, rows=128, claims=('many', 'straddle', 'short_last'))),
    ('logp_f32_v1027_s1500_c128', _c('logp', F32, 2, 1500, 1027, rows=128,
                                     claims=('many', 'straddle', 'short_last', 'long_seq'))),
    ('logp_f32_v56324_s127_c128', _c('logp', F32, 2, 127, 56324, rows=128, claims=('straddle', 'short_last'))),
    ('logp_f32_v152063_r3', _c('logp', F32, 1, 3, 152063, claims=('one', ))),
    ('logp_bf16_v7_b1104_c1024', _c('logp', BF16, 1104, 2, 7, rows=1024, claims=('loop', ))),
    ('logp_bf16_v1003_one', _c('logp', BF16, 4, 75, 1003, claims=('one', ))),
    ('logp_bf16_v112648_s129_c128', _c('logp', BF16, 2, 129, 112648, rows=128, claims=('many', 'straddle', 'short_last'))),
    ('logp_bf16_v152064_r3', _c('logp', BF16, 3, 1, 152064, claims=('one', ))),
])
UPSTREAMS = (0.37, -2.0, 0.0)
NEEDS = ((True, False), (False, True), (True, True))  # hidden, lm_weight requiring grad on the g != 1 paths


def _esize(c):
    return 4 if c['dtype'] == F32 else 2


def _budget(c):
    return c['rows'] * c['V'] * _esize(c) if c['rows'] else 1 << 30


@contextlib.contextmanager
def _plan_budget(nbytes):
    saved = ops.LM_CHUNK_BYTES
    ops.LM_CHUNK_BYTES = nbytes
    try:
        yield
    finally:
        ops.LM_CHUNK_BYTES = saved


def plan(c, sms=SMS):
    """(rows per chunk, chunks) of the case's call"""
    with _plan_budget(_budget(c)):
        return ops.lm_chunk_plan(c['B'] * c['S'], c['V'], _esize(c), sms, c['kind'] != 'logp',
                                 5 if c['kind'] == 'ppo' else 3)


def _names(c):
    if c['names']:
        return c['names']
    if c['kind'] == 'grpo' or (c['kind'] == 'ppo' and c['kl']):
        return vf.REGIMES
    return vf.REGIMES[:-1] if c['kind'] in ('rloo', 'ppo') else NO_OLD


# ----------------------------------------------------------------------------------------------------------------
# the generator (CPU)
# ----------------------------------------------------------------------------------------------------------------
def gen_case(name):
    """-> dict: Zr (R, V) logit rows, idx (N) the logit row of each token, action (N), lp_old / lp_ref (N) fp32 or None,
    weight, adv / reward / value / return_, onpolicy (N) bool, meta (regime per token)"""
    c = CASES[name]
    B, S, V, dtype = c['B'], c['S'], c['V'], c['dtype']
    N = B * S
    seed = 12000 + list(CASES).index(name)
    kind = c['kind']
    names = _names(c)
    with_ref = kind == 'grpo' or (kind == 'ppo' and c['kl'] is not None)
    rows, _ = plan(c)
    R = P_PERIOD if c['periodic'] else N
    new, old, ref, act_r, meta = vf.gen_rows(seed, R, V, dtype, names, with_ref, MASKS, rows)
    idx = torch.arange(N) % R
    action = act_r[idx]
    g = torch.Generator().manual_seed(seed + 1)
    out = dict(Zr=new, idx=idx, action=action, weight=vf._weights(g, B, S, c['w'], zero_seq=c['zero']),
               meta=dict(regime=meta['regime'][idx.numpy()], names=meta['names']))
    out['onpolicy'] = torch.from_numpy(out['meta']['regime'] == list(names).index('onpolicy')) if 'onpolicy' in names \
        else torch.zeros(N, dtype=torch.bool)
    out['lp_old'] = go.logp64(old[idx], action, F32) if kind in ('grpo', 'rloo', 'ppo') else None
    out['lp_ref'] = go.logp64(ref[idx], action, F32) if with_ref else None
    if c['periodic']:  # per-token log-probabilities: the tokens that share a logit row differ in their ratios
        for k in ('lp_old', 'lp_ref'):
            if out[k] is not None:
                out[k] = out[k] + 0.01 * torch.randn(N, generator=g)
    if kind == 'grpo':
        out['adv'] = torch.randn(B, generator=g)
        out['adv'][::7] = 0.0
    elif kind == 'rloo':
        out['reward'] = vf._rewards(g, c['K'], B // c['K'])
    elif kind == 'ppo':
        out['adv'] = vf.a2c_side(g, B, S)[0]
    elif kind == 'a2c':
        out['adv'], out['return_'], out['value'] = vf.a2c_side(g, B, S)
    if kind == 'logp':
        up = torch.randn(N, generator=g)
        up[torch.rand(N, generator=g) < 0.1] = 0.0
        up[:4] = torch.tensor([0.37, -2.0, 0.0, vf.NEXT1])[:N]
        out['up'] = up.reshape(B, S)
    return out


def one_hot_inputs(Zr, idx, periodic):
    """(H (N, D), W (V, D)) with F.linear(H, W) = Zr[idx]: D = N and H = I, or D = P and H row n = e_(n mod P)"""
    N = idx.numel()
    D = Zr.shape[0] if periodic else N
    H = torch.zeros(N, D, dtype=Zr.dtype, device=Zr.device)
    H[torch.arange(N, device=Zr.device), idx.to(Zr.device) if periodic else torch.arange(N, device=Zr.device)] = 1
    W = (Zr if periodic else Zr[idx.to(Zr.device)]).t().contiguous()
    return H, W


# ----------------------------------------------------------------------------------------------------------------
# references
# ----------------------------------------------------------------------------------------------------------------
def refs(c, d, Z, lp_old, up=None, dtype=torch.float64):
    """scalars and dZ (N, V) [and d value (N)] of the case for a unit upstream gradient of the one loss (log p: the
    per-token upstream ``up``), in ``dtype``"""
    B, S, V = c['B'], c['S'], c['V']
    kind = c['kind']
    a = d['action']
    if kind == 'logp':
        return OrderedDict(lp=vf._np(go.logp64(Z, a, dtype))), go.grad_rows64(Z, a, up.reshape(-1).to(dtype), dtype), None
    if kind in ('grpo', 'rloo'):
        dd = {'logit_new': Z.reshape(B, S, V), 'action': a.reshape(B, S), 'weight': d['weight']}
        dd.update({'adv': d['adv']} if kind == 'grpo' else {'reward': d['reward']})
        r = go.run64(dd, dtype=dtype, lp_old=lp_old, lp_ref=d['lp_ref'])
        out = OrderedDict([('out_loss', r['loss']), ('out_approx_kl', r['approx_kl']), ('out_clipfrac', r['clipfrac'])])
        return out, go.grad_rows64(Z, a, r['dlp'].reshape(-1), dtype), None
    if kind == 'ppo':
        dd = {'logit_new': Z.reshape(B, S, V), 'action': a.reshape(B, S), 'weight': d['weight'], 'adv': d['adv']}
        mix = (1.0, -EW if c['ent'] else 0.0, KW if c['kl'] else 0.0)
        r = po.run64(dd, dual_clip=c['dc'], kl_type=c['kl'] or 'k1', entropy_bonus=c['ent'], mix=mix, dtype=dtype,
                     lp_old=lp_old, lp_pre=d['lp_ref'])
        loss = torch.tensor(r['policy'], dtype=dtype)
        if c['ent']:
            loss = loss + mix[1] * r['entropy']
        if c['kl']:
            loss = loss + mix[2] * r['kl']
        out = OrderedDict([('out_loss', loss.item()), ('out_policy', r['policy']), ('out_entropy', r['entropy']),
                           ('out_kl', r['kl']), ('out_approx_kl', r['approx_kl']), ('out_clipfrac', r['clipfrac'])])
        return out, r['grad'].reshape(-1, V), None
    x = Z.reshape(B, S, V).to(dtype, copy=True).requires_grad_(True)
    v = d['value'].to(dtype, copy=True).requires_grad_(True)
    w = None if d['weight'] is None else d['weight'].to(dtype)
    p, vl, e = rl_oracle.a2c_error(x, a.reshape(B, S), v, d['adv'].to(dtype), d['return_'].to(dtype), w)
    loss = p + VW * vl - EW * e
    loss.backward()
    out = OrderedDict([('out_loss', loss.item()), ('out_policy', p.item()), ('out_value', vl.item()),
                       ('out_entropy', e.item())])
    return out, x.grad.reshape(-1, V), v.grad.reshape(-1)


def meta64(c, d, Z, lp_old):
    """(boundary rows, loss scales, per-row scale of dZ for a unit upstream gradient) in float64"""
    kind = c['kind']
    N = Z.shape[0]
    a = d['action']
    Zd = Z.double()
    lse = torch.logsumexp(Zd, -1)
    za = Zd.gather(-1, a.unsqueeze(-1)).squeeze(-1)
    lpn = (za - lse).cpu().numpy()
    B, S = c['B'], c['S']
    w = np.ones(N) if d['weight'] is None else d['weight'].double().reshape(-1).cpu().numpy()
    if kind == 'logp':
        return None, {}, np.abs(d['up'].double().reshape(-1).cpu().numpy())
    lsm = torch.log_softmax(Zd, -1)
    H = -(torch.exp(lsm) * lsm).nan_to_num(0.0).sum(-1).cpu().numpy()
    if kind == 'a2c':
        adv = d['adv'].double().reshape(-1).cpu().numpy()
        dv = (d['return_'] - d['value']).double().reshape(-1).cpu().numpy()
        scales = {'out_policy': np.mean(np.abs(lpn * adv * w)), 'out_value': np.mean(dv ** 2 * w),
                  'out_entropy': np.mean(np.abs(H * w))}
        scales['out_loss'] = scales['out_policy'] + VW * scales['out_value'] + EW * scales['out_entropy']
        return None, scales, (w * np.abs(adv) + EW * w * (1 + H)) / N
    lpo = lp_old.double().reshape(-1).cpu().numpy()
    ratio = np.exp(lpn - lpo)
    lse_sz = np.abs(lse.cpu().numpy()) + np.abs(za.cpu().numpy()) + np.abs(lpo)
    if kind in ('grpo', 'rloo'):
        adv = (d['adv'].double().cpu() if kind == 'grpo' else go.rloo_adv64(d['reward'].cpu())).numpy()
        adv_r = np.repeat(adv, S)
        with np.errstate(invalid='ignore', divide='ignore'):
            wn = (w.reshape(B, S) / w.reshape(B, S).sum(1, keepdims=True)).reshape(-1)
        tok = np.abs(np.minimum(ratio * adv_r, np.clip(ratio, 1 - go.CLIP, 1 + go.CLIP) * adv_r))
        if kind == 'grpo':
            dr = d['lp_ref'].double().reshape(-1).cpu().numpy() - lpn
            tok = tok + go.BETA * np.abs(np.exp(dr) - dr - 1)
        scales = {'out_loss': float(np.nansum(tok * wn)) / B, 'out_approx_kl': float(np.mean(np.abs(lpo - lpn)))}
        return vf._boundary(ratio, adv_r, lse_sz), scales, None  # the row scale is run64's
    adv = d['adv'].double().reshape(-1).cpu().numpy()
    _, _, pol = policy_terms(ratio, adv, w, np.ones(N), go.CLIP, c['dc'])
    scales = {'out_policy': pol, 'out_approx_kl': float(np.mean(np.abs(lpo - lpn)))}
    row = w * np.abs(adv) * ratio
    loss_sc = pol
    if c['ent']:
        scales['out_entropy'] = float(np.mean(np.abs(H * w)))
        row = row + EW * w * (1.0 + H)
        loss_sc += EW * scales['out_entropy']
    if c['kl']:
        lr = lpn - d['lp_ref'].double().reshape(-1).cpu().numpy()
        kt = {'k1': lr, 'k2': lr ** 2 / 2, 'k3': np.exp(-lr) - 1 + lr}[c['kl']]
        scales['out_kl'] = float(np.mean(np.abs(kt)))
        row = row + KW * (1.0 + np.abs(lr) + np.exp(-lr))
        loss_sc += KW * scales['out_kl']
    scales['out_loss'] = loss_sc
    return vf._boundary(ratio, adv, lse_sz, c['dc']), scales, row / N


# ----------------------------------------------------------------------------------------------------------------
# the calls
# ----------------------------------------------------------------------------------------------------------------
def call(c, d, h, w, v=None):
    """-> (the differentiable output, OrderedDict of its scalars / per-token lp, d value's owner or None)"""
    import di_engine_b200 as b2
    R = b2.rl_utils
    B, S = c['B'], c['S']
    h = h.reshape(B, S, -1)
    kind = c['kind']
    if kind == 'logp':
        lp = R.token_logp_linear(h, w, d['action'].reshape(B, S))
        return lp, OrderedDict(lp=lp.detach().reshape(-1).double().cpu().numpy())
    if kind in ('grpo', 'rloo'):
        a = d['action'].reshape(B, S)
        lpo = d['lp_old'].reshape(B, S)
        if kind == 'grpo':
            loss, info = R.grpo_policy_error_linear(R.grpo_linear_data(h, w, lpo, d['lp_ref'].reshape(B, S), a, d['adv'],
                                                                       d['weight']), go.CLIP, go.BETA)
        else:
            loss, info = R.rloo_policy_error_linear(R.rloo_linear_data(h, w, lpo, a, d['reward'], d['weight']), go.CLIP)
        return loss, OrderedDict([('out_loss', loss.item()), ('out_approx_kl', info.approx_kl),
                                  ('out_clipfrac', info.clipfrac)])
    if kind == 'ppo':
        lpp = None if d['lp_ref'] is None else d['lp_ref'].reshape(B, S)
        out, info = R.ppo_policy_error_linear(
            R.ppo_policy_linear_data(h, w, d['lp_old'].reshape(B, S), d['action'].reshape(B, S), d['adv'], d['weight'],
                                     lpp), go.CLIP, c['dc'], c['ent'], c['kl'] or 'k1', EW if c['ent'] else 0.0,
            KW if c['kl'] else 0.0)
        return out.loss, OrderedDict([('out_loss', out.loss.item()), ('out_policy', out.policy_loss.item()),
                                      ('out_entropy', out.entropy_loss.item()), ('out_kl', out.kl_div.item()),
                                      ('out_approx_kl', info.approx_kl), ('out_clipfrac', info.clipfrac)])
    out = R.a2c_error_linear(R.a2c_linear_data(h, w, d['action'].reshape(B, S), v, d['adv'], d['return_'], d['weight']),
                             VW, EW)
    return out.loss, OrderedDict([('out_loss', out.loss.item()), ('out_policy', out.policy_loss.item()),
                                  ('out_value', out.value_loss.item()), ('out_entropy', out.entropy_loss.item())])


def run(c, d, H, W, needs, g=1.0, twice=False, grad=True):
    """one call and backward of (out * g) ['twice': a second backward through the same graph, the recompute path];
    -> (scalars, dH, dW, d value)"""
    h = H.clone().requires_grad_(needs[0])
    w = W.clone().requires_grad_(needs[1])
    v = None
    if c['kind'] == 'a2c':
        v = d['value'].clone().requires_grad_(len(needs) > 2 and needs[2])
    ctx = contextlib.nullcontext() if grad else torch.no_grad()
    with ctx:
        out, res = call(c, d, h, w, v)
    if grad and out.requires_grad:
        if c['kind'] == 'logp':
            y = (out * (d['up'] * g)).sum()
        else:
            y = out * g if g != 1.0 else out
        y.backward(retain_graph=twice)
        if twice:
            y.backward()
    return res, h.grad, w.grad, None if v is None else v.grad


# ----------------------------------------------------------------------------------------------------------------
# GPU
# ----------------------------------------------------------------------------------------------------------------
@pytest.fixture
def exact_gemm(monkeypatch):
    """fp32 GEMMs in fp32 (no TF32) and bf16 GEMMs reduced in fp32: F.linear(I, Z^T) is then Z bit for bit"""
    monkeypatch.setattr(torch.backends.cuda.matmul, 'allow_tf32', False)
    monkeypatch.setattr(torch.backends.cuda.matmul, 'allow_bf16_reduced_precision_reduction', False)


class Case:
    pass


@functools.lru_cache(maxsize=1)
def _case(name):
    c = CASES[name]
    cs = Case()
    cs.c = c
    d = gen_case(name)
    meta = d.pop('meta')
    d = {k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in d.items()}
    cs.meta = meta
    H, W = one_hot_inputs(d['Zr'], d['idx'], c['periodic'])
    Z = d['Zr'][d['idx']]
    # the construction checks itself: the GEMM the chunk loop runs gives the logits bit for bit
    assert torch.equal(F.linear(H, W), Z), name
    if d['onpolicy'].any():  # logp_old of the on-policy rows: the first step of every GRPO / PPO iteration
        with torch.no_grad():
            lp_on = ops.lm_logp_fwd_(H, W, d['action'], ops._LOGIT_DTYPES[c['dtype']])[0]
        d['lp_old'] = torch.where(d['onpolicy'], lp_on, d['lp_old'])
    cs.d, cs.H, cs.W, cs.Z = d, H, W, Z
    cs.r = {}
    for dt in (torch.float64, torch.float32):
        cs.r[dt] = refs(c, d, Z, d['lp_old'], d.get('up'), dt)
    cs.bnd, cs.scales, row = meta64(c, d, Z, d['lp_old'])
    if row is None:  # GRPO / RLOO: run64's scale
        dd = {'logit_new': Z.reshape(c['B'], c['S'], -1), 'action': d['action'].reshape(c['B'], c['S']),
              'weight': d['weight']}
        dd.update({'adv': d['adv']} if c['kind'] == 'grpo' else {'reward': d['reward']})
        row = go.run64(dd, lp_old=d['lp_old'], lp_ref=d['lp_ref'])['scale'].reshape(-1).cpu().numpy()
    cs.div = vf.row_divisor(row)
    return cs


def _drop_out_of_range(a, b, *xs):
    """zero, in every numpy array xs, the entries of the GEMM a @ b where |a| @ |b| passes float32's range: there a
    float32 GEMM may give inf, or NaN from partial sums of both signs, whatever its order (the construction's W holds the
    masked regime's -1e30 logits, and a large-regime gradient row times them leaves that range)"""
    oor = vf._np(a.abs() @ b.abs()) > torch.finfo(torch.float32).max
    assert oor.mean() < 0.01, oor.mean()
    for x in xs:
        x[oor] = 0.0


def check_unit(cs, tag, res, dh, dw, dv, full=True):
    """the K bound for the scalars, lp, dZ (through dW), dH, the periodic dW and d value of a unit upstream gradient"""
    c, d = cs.c, cs.d
    bf16 = c['dtype'] == BF16
    div = cs.div
    exact_dz = not c['periodic'] and not c['zero']
    got, r32, r64 = OrderedDict(res), OrderedDict(cs.r[torch.float32][0]), OrderedDict(cs.r[torch.float64][0])
    for k in list(r64):
        if k in ('out_entropy', 'out_kl') and not c[{'out_entropy': 'ent', 'out_kl': 'kl'}[k]] and c['kind'] == 'ppo':
            assert got[k] == 0.0, (tag, k)
            for x in (got, r32, r64):
                x.pop(k)
    dz64, dz32 = cs.r[torch.float64][1], cs.r[torch.float32][1]
    if full and dw is not None and exact_dz:
        want64 = vf._np(dz64)
        got['grad_dz'] = vf.grad_entry(dw.t(), div, bf16, want64)
        r64['grad_dz'] = want64 / div[:, None]
        r32['grad_dz'] = vf._np(dz32) / div[:, None]
    if full and dh is not None:
        W64 = cs.W.double()
        if bf16:  # the kernel's own dZ (checked above) through float64 and through the same bf16 GEMM, unchunked
            assert exact_dz and dw is not None, 'bf16 cases are exact, without a zero-weight sequence'
            h64, h32 = dw.t().double() @ W64, torch.mm(dw.t(), cs.W)
        else:
            h64, h32 = dz64 @ W64, dz32 @ cs.W
        want = vf._np(h64)
        got['grad_dh'] = vf.grad_entry(dh.reshape(len(div), -1), div, False)
        r64['grad_dh'] = want / div[:, None]
        r32['grad_dh'] = vf._np(h32) / div[:, None]
        _drop_out_of_range(dz64 if not bf16 else dw.t().double(), W64, got['grad_dh'], r64['grad_dh'], r32['grad_dh'])
    if dv is not None:
        got['grad_value'] = vf._np(dv.reshape(-1))
        r64['grad_value'] = vf._np(cs.r[torch.float64][2])
        r32['grad_value'] = vf._np(cs.r[torch.float32][2])
    worst = vf.compare_regimes(tag, got, r32, r64, cs.meta, cs.scales, cs.bnd)
    if full and dw is not None and not exact_dz:  # dW as a tensor: a sum of N / P gradient rows, or NaN throughout
        H64 = cs.H.double()
        w64, w32 = dz64.t() @ H64, dz32.t() @ cs.H.float()
        x, a, b = vf._np(dw), vf._np(w32), vf._np(w64)
        _drop_out_of_range(dz64.t(), H64, x, a, b)
        worst = max(worst, compare64(tag + ' dW', OrderedDict(grad_dw=x), OrderedDict(grad_dw=a), OrderedDict(grad_dw=b)))
    return worst


def _scaled(x, g):
    return None if x is None else (x.float() * g).to(x.dtype)


@pytest.mark.gpu
@pytest.mark.parametrize('name', list(CASES))
def test_lm_linear_fp64(name, exact_gemm, monkeypatch):
    monkeypatch.setattr(ops, 'LM_CHUNK_BYTES', _budget(CASES[name]))
    cs = _case(name)
    c, d = cs.c, cs.d
    a2c = c['kind'] == 'a2c'
    vf.WORST.clear()
    torch.cuda.reset_peak_memory_stats()
    both = (True, True, True) if a2c else (True, True)
    # the forward alone (no row cache, no gradient buffer)
    res = run(c, d, cs.H, cs.W, both, grad=False)[0]
    worst = check_unit(cs, name + ' nograd', res, None, None, None, full=False)
    # a unit upstream gradient, every input requiring grad: the forward-written gradients
    unit = run(c, d, cs.H, cs.W, both)
    worst = max(worst, check_unit(cs, name + ' unit', *unit))
    if c['names'] == ('onpolicy', ):
        assert unit[0]['out_clipfrac'] == 0.0
    # the same plan repeats bit for bit
    again = run(c, d, cs.H, cs.W, both)
    for k in unit[0]:
        np.testing.assert_array_equal(again[0][k], unit[0][k])  # NaN where NaN
    for x, y in zip(again[1:], unit[1:]):
        assert (x is None and y is None) or torch.equal(x.nan_to_num(7.0), y.nan_to_num(7.0)), name
    # upstream gradients != 1: exactly the unit gradients scaled in place, for each input alone and both
    i = list(CASES).index(name)
    logp = c['kind'] == 'logp'  # its backward takes the per-token upstream itself: g = 1, each input alone and both
    for k, g in enumerate((1.0, 1.0, 1.0) if logp else (vf.NEXT1, UPSTREAMS[i % 3], UPSTREAMS[(i + 1) % 3])):
        needs = NEEDS[(i + k) % 3] + ((k % 2 == 0, ) if a2c else ())
        got = run(c, d, cs.H, cs.W, needs, g)
        for x, y, need in zip(got[1:], unit[1:], needs):
            if not need:
                assert x is None
            else:
                assert torch.equal(x.nan_to_num(7.0), _scaled(y, g).nan_to_num(7.0)), (name, g, needs)
        if c['dtype'] == F32 and g == vf.NEXT1 and got[1] is not None:
            nz = unit[1].abs() >= torch.finfo(F32).tiny  # a subnormal times nextafter(1, 2) rounds back to itself
            assert (got[1][nz] != unit[1][nz]).all(), 'the nextafter(1, 2) scale was skipped'
    # a repeated backward: the recompute path, bit for bit 2 * the scaled unit gradients
    g = 1.0 if logp else UPSTREAMS[i % 3]
    got = run(c, d, cs.H, cs.W, both, g, twice=True)
    for x, y in zip(got[1:], unit[1:]):
        if y is not None:
            assert torch.equal(x.nan_to_num(7.0), (_scaled(y, g) * 2).nan_to_num(7.0)), (name, 'twice')
    if a2c:  # value alone: the chunk kernel gets no gradient buffer and still writes d value
        got = run(c, d, cs.H, cs.W, (False, False, True))
        assert got[1] is None and got[2] is None and torch.equal(got[3], unit[3])
    # another chunk plan: within the bound
    if c['rows']:
        monkeypatch.setattr(ops, 'LM_CHUNK_BYTES', 1 << 30)
        other = run(c, d, cs.H, cs.W, both)
        worst = max(worst, check_unit(cs, name + ' one chunk', *other))
    print('[fp64] %s worst %.2f  per regime %s  peak %.0f MiB' % (name, worst, vf._per_regime(),
                                                                  torch.cuda.max_memory_allocated() / 2 ** 20))


OVERFLOW = {'grpo_f32': ('grpo', F32), 'grpo_bf16': ('grpo', BF16), 'ppo_f32': ('ppo_kl', F32),
            'ppo_bf16': ('ppo_kl', BF16)}


@pytest.mark.gpu
@pytest.mark.parametrize('name', list(OVERFLOW))
def test_overflow_rows_match_the_fp32_pattern(name, exact_gemm):
    """rows whose ratio overflows fp32 (not fp64): test_vocab_fp64's overflow regime, its logp_old given per token"""
    kind, dtype = OVERFLOW[name]
    d, ov = vf._overflow_case(vf.OVERFLOW_SEEDS[name], dtype, kind)
    B, S, V = d['logit_new'].shape
    c = _c('grpo' if kind == 'grpo' else 'ppo', dtype, B, S, V, 'frac', ent=kind != 'grpo', kl='k3' if kind != 'grpo'
           else None, dc=None if kind == 'grpo' else 2.0)
    a = d['action'].reshape(-1)
    dd = {'action': a.to(DEV), 'weight': d['weight'].to(DEV), 'lp_old': go.logp64(d['logit_old'].reshape(-1, V), a, F32)}
    ref = d['logit_ref'] if kind == 'grpo' else d['logit_pretrained']
    dd['lp_ref'] = go.logp64(ref.reshape(-1, V), a, F32)
    dd.update({'adv': d['adv'].to(DEV)})
    dd = {k: v.to(DEV) for k, v in dd.items()}
    Z = d['logit_new'].reshape(-1, V).to(DEV)
    H, W = one_hot_inputs(Z, torch.arange(B * S), False)
    assert torch.equal(F.linear(H, W), Z)
    r32, dz32, _ = refs(c, dd, Z, dd['lp_old'], None, F32)
    res, dh, dw, _ = run(c, dd, H, W, (True, True))
    assert not torch.isfinite(dz32[torch.from_numpy(ov).to(DEV)]).all()
    for k in r32:
        x, b = np.float64(res[k]), np.float64(r32[k])
        assert np.isnan(x) == np.isnan(b) and np.isposinf(x) == np.isposinf(b) and np.isneginf(x) == np.isneginf(b), \
            (name, k, x, b)
    # dW mixes every row into every entry (inf * 0 is NaN); dH row n is non-finite exactly where dZ row n is
    assert torch.equal(torch.isfinite(dh.reshape(B * S, -1)).all(1), torch.isfinite(dz32).all(1)), name
    assert not torch.isfinite(dh.reshape(B * S, -1)).all(1)[torch.from_numpy(ov).to(DEV)].all()


# ----------------------------------------------------------------------------------------------------------------
# dense hidden states at D's edges, a strided hidden and a transposed lm_weight (test_lm_linear's composition rule)
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('dtype', [F32, BF16])
@pytest.mark.parametrize('D', [1, 63, 4096])
@pytest.mark.parametrize('kind', ['grpo', 'rloo'])
def test_dense_hidden_at_d_edges(monkeypatch, kind, D, dtype):
    from tests import test_lm_linear as tl
    monkeypatch.setattr(ops, 'LM_CHUNK_BYTES', 128 * 1003 * 4)
    d = tl.gpu_case(kind, dtype, 4, 75, D, 1003, seed=D)
    got = tl.compare(kind, d)
    # the same hidden states as a slice of a (B, S, 2D) tensor, and the weight stored transposed: _stage's copies map the
    # gradients back, bit for bit those of the contiguous call
    wide = torch.cat([d['hidden'], torch.randn_like(d['hidden'].float()).to(dtype)], -1).requires_grad_(True)
    wt = d['lm_weight'].t().contiguous().requires_grad_(True)
    assert not wide[..., :D].is_contiguous() or D == 1
    loss, info = tl.loss_call(kind, dict(d, hidden=wide[..., :D], lm_weight=wt.t()), clip_ratio=go.CLIP,
                              **({'beta': go.BETA} if kind == 'grpo' else {}))
    loss.backward()
    assert loss.item() == got[0] or (math.isnan(got[0]) and math.isnan(loss.item()))
    assert torch.equal(wide.grad[..., :D], got[3]) and not wide.grad[..., D:].any()
    assert torch.equal(wt.grad.t(), got[4])


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', [F32, BF16])
@pytest.mark.parametrize('D', [1, 63, 4096])
def test_dense_hidden_at_d_edges_ppo_a2c(monkeypatch, D, dtype):
    """ppo_policy_error_linear and a2c_error_linear at the same D, against the composition and float64"""
    from tests import test_lm_linear_pg as tp
    monkeypatch.setattr(ops, 'LM_CHUNK_BYTES', 128 * 1003 * 4)
    for kind in ('ppo', 'a2c'):
        tp.compare(kind, tp.gpu_case(dtype, 4, 75, D, 1003, seed=D, pre=kind == 'ppo'),
                   (2.0, 'k3', True) if kind == 'ppo' else None)


# ----------------------------------------------------------------------------------------------------------------
# CPU: the construction, the comparison's teeth and the hand-off claims of the table
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('periodic', [False, True])
def test_one_hot_identity_fp32_on_cpu(periodic):
    new, _, _, action, meta = vf.gen_rows(12500, 600 if periodic else 257, 1027, F32, vf.REGIMES, True, MASKS, 128)
    assert torch.isfinite(new).all() and (new[meta['mask']] <= -1e4).all()
    idx = torch.arange(1200 if periodic else 257) % new.shape[0]
    if periodic:
        new = new[:P_PERIOD]
        idx = torch.arange(1200) % P_PERIOD
    H, W = one_hot_inputs(new, idx, periodic)
    assert torch.equal(F.linear(H, W), new[idx])
    assert torch.equal(torch.mm(H[:128], W.t()), new[idx[:128]])  # one chunk's GEMM, as lm_chunks_ runs it
    dz = torch.randn(idx.numel(), 1027)
    if not periodic:
        assert torch.equal(dz.t() @ H, dz.t())  # dW is dZ^T bit for bit


def _cpu_case():
    """a small exact GRPO case on the CPU: refs in float64 / float32, the per-row divisors and meta"""
    c = _c('grpo', F32, 3, 100, 300, 'frac', rows=128)
    new, old, ref, action, meta = vf.gen_rows(12600, 300, 300, F32, vf.REGIMES, True, MASKS, 128)
    g = torch.Generator().manual_seed(5)
    d = {'action': action, 'weight': vf._weights(g, 3, 100, 'frac'), 'adv': torch.randn(3, generator=g),
         'lp_old': go.logp64(old, action, F32), 'lp_ref': go.logp64(ref, action, F32)}
    r64 = refs(c, d, new, d['lp_old'])
    r32 = refs(c, d, new, d['lp_old'], dtype=F32)
    dd = {'logit_new': new.reshape(3, 100, 300), 'action': action.reshape(3, 100), 'weight': d['weight'],
          'adv': d['adv']}
    div = vf.row_divisor(go.run64(dd, lp_old=d['lp_old'], lp_ref=d['lp_ref'])['scale'].reshape(-1).numpy())
    return new, r64, r32, div, meta


def test_regime_checks_are_real_through_dw():
    """the comparison of dZ read through dW rejects one corrupted element, one row left as stale logits and two rows
    swapped across the chunk boundary at row 128"""
    Z, r64, r32, div, meta = _cpu_case()
    want64 = r64[1].numpy()
    R32 = OrderedDict(grad_dz=r32[1].double().numpy() / div[:, None])
    R64 = OrderedDict(grad_dz=want64 / div[:, None])
    H, W = one_hot_inputs(Z, torch.arange(300), False)

    def check(dz):
        dw = dz.t().contiguous() @ H  # the dW the chunk loop returns, read back as the kernel's dZ
        vf.compare_regimes('dz', OrderedDict(grad_dz=vf.grad_entry(dw.t(), div, False, want64)), R32, R64, meta)

    good = r32[1].clone()
    check(good)
    worst_row = int(np.argmax(np.abs(want64).max(1) / div))
    for bad in ('element', 'stale', 'swap'):
        dz = good.clone()
        if bad == 'element':
            r = int(np.argmin(div))  # the row with the smallest coefficient: the whole-tensor scale would hide it
            v = int(np.abs(want64[r]).argmax())
            dz[r, v] += 1e-3 * float(div[r])
        elif bad == 'stale':
            r = worst_row
            dz[r] = Z[r]
        else:
            dz[[127, 128]] = dz[[128, 127]]
        with pytest.raises(AssertionError):
            check(dz)


def _claims(c, sms=SMS):
    rows, n = plan(c, sms)
    N, S = c['B'] * c['S'], c['S']
    last = N - (n - 1) * rows
    sums = 5 if c['kind'] == 'ppo' else 3
    grid_max = min(rows, sms * ops._VOCAB_CTAS_PER_SM)
    out = set()
    if n == 1:
        out.add('one')
    if n >= 3 and rows == 128:
        out.add('many')
    if rows > grid_max:
        out.add('loop')  # more rows than any grid of the chunk kernel: a CTA owns several rows of a chunk
    if n > 1 and last < min(rows, sms):
        out.add('short_last')  # the grid is at least min(rows, SMs): idle CTAs in the last chunk
    if c['kind'] != 'logp' and (n + 1) * grid_max * sums > ops._WS_PARTIAL_WORDS:
        out.add('limit')  # no further chunk's partials would fit
    if any((k * rows) % S for k in range(1, n)):
        out.add('straddle')
    if S > 256 and S > 10 * rows:
        out.add('long_seq')  # more than lm_seq_kernel's 256 threads, across more than 10 chunks
    if c['B'] > sms * LM_SEQ_PER_SM:
        out.add('b_grid')
    return out


@pytest.mark.parametrize('name', list(CASES))
def test_case_claims_hold_at_132_sms(name):
    c = CASES[name]
    got = _claims(c)
    assert c['claims'] <= got, (name, sorted(c['claims'] - got))
    N = c['B'] * c['S']
    assert c['periodic'] or N * N * _esize(c) <= 64 << 20, 'the exact construction holds an N x N identity'
    if c['periodic']:
        assert c['dtype'] == F32 and N > P_PERIOD


def test_the_table_reaches_every_hand_off():
    claims = set().union(*(c['claims'] for c in CASES.values()))
    assert claims == {'one', 'many', 'loop', 'short_last', 'limit', 'straddle', 'long_seq', 'b_grid'}
    vs = {(c['dtype'], c['V']) for c in CASES.values()}
    assert {(F32, V) for V in (1, 3, 1027, 56320, 56324, 152063)} <= vs
    assert {(BF16, V) for V in (1, 7, 1003, 112640, 112648, 152064)} <= vs
    for kind in ('grpo', 'rloo', 'ppo', 'a2c', 'logp'):
        assert any(c['kind'] == kind and c['claims'] & {'many'} for c in CASES.values()), kind
    assert {c['K'] for c in CASES.values() if c['kind'] == 'rloo'} >= {2, 3, 64}
    assert any(c['kind'] == 'rloo' and c['K'] == c['B'] for c in CASES.values())
    assert {(c['ent'], c['kl'], c['dc']) for c in CASES.values() if c['kind'] == 'ppo'} >= {
        (e, k, dc) for e in (False, True) for k in (None, 'k1', 'k2', 'k3') for dc in (None, 2.0)}
    assert {c['w'] for c in CASES.values()} == {None, 'mask', 'frac'}
    assert any(c['S'] == 1 for c in CASES.values()) and any(c['S'] >= 1500 for c in CASES.values())
    assert {127, 128, 129} & {c['S'] for c in CASES.values()} >= {127, 129}
    # the largest plan: its last chunk's partials end within one chunk's slice of the workspace's end
    c = CASES['ppo_f32_v1027_limit_ent_k3_dc']
    rows, n = plan(c)
    assert (rows, n) == (128, PPO_LIMIT_CHUNKS) and ops._WS_PARTIAL_WORDS - n * 128 * 5 < 128 * 5
    with _plan_budget(_budget(c)), pytest.raises(ValueError, match='partials'):
        ops.lm_chunk_plan((n + 1) * 128, c['V'], 4, SMS, True, 5)


def test_largest_plan_launches(monkeypatch):
    """the recording stand-in: the largest PPO plan launches its 399 chunks at row0 = 0, 128, ..., 398 * 128, all with the
    same chunk size and N, and the loss sums of the last"""
    from tests.test_lm_linear import _RecordingLib
    from tests.test_lm_linear_pg import A_CHUNK, A_N, A_ROW0, A_ROWS
    rec = _RecordingLib()
    monkeypatch.setattr(ops, 'lib', lambda: rec)
    monkeypatch.setattr(ops, 'require_cuda', lambda: None)
    monkeypatch.setattr(ops, 'compute_device', lambda *t: torch.device('cpu'))
    monkeypatch.setattr(ops, 'stream_ptr', lambda: 0)
    monkeypatch.setattr(ops, 'sm_count', lambda dev: SMS)
    monkeypatch.setattr(torch.cuda, 'device', lambda d: contextlib.nullcontext())
    monkeypatch.setattr(ops, 'LM_CHUNK_BYTES', 128 * 3 * 4)
    ops._WS.clear()
    import di_engine_b200 as b2
    R = b2.rl_utils
    B, S = 32, PPO_LIMIT_CHUNKS * 4
    N = B * S
    try:
        h = torch.zeros(B, S, 2)
        w = torch.zeros(3, 2)
        z = torch.zeros(B, S)
        with torch.no_grad():
            R.ppo_policy_error_linear(R.ppo_policy_linear_data(h, w, z, z.long(), z, None, z), kl_type='k3')
    finally:
        ops._WS.clear()
    fwd = [c[1] for c in rec.calls if c[0] == 'b200rl_lm_linear_pg_fwd']
    assert [(f[A_ROW0], f[A_ROWS], f[A_CHUNK], f[A_N]) for f in fwd] == [(k * 128, 128, 128, N)
                                                                         for k in range(PPO_LIMIT_CHUNKS)]
