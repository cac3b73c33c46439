"""The vocabulary-scale kernels of csrc/vocab.cu against a float64 reference, on token rows where an online softmax goes
wrong.

Kernels: ``vocab_rows_kernel<T, Head>`` for fp32 and bf16 logits -- grpo_policy_error, rloo_policy_error (GrpoRow with
and without the cached row, CoefBwdRow), the three log-prob methods (LogpRow, CoefBwdRow) and language-model
ppo_policy_error (PpoRow with its entropy / KL flags, PgBwdRow), language-model a2c_error (A2cRow, backward PgBwdRow with
the value slot, on the regimes without an old policy, returns at 1e3 with a 1e-2 spread, value == return and adv = 0,
each mix from the record with the forward's gradient buffers poisoned: a mix that differs only in the value slot keeps
d logit and rewrites d value) -- and ``token_head_kernel`` (a custom log_prob_fn).

The seeded parity cases of test_grpo_rloo.py / test_ppo_lm.py draw ``logit_old = new + 0.1 randn`` and logit scales of
1..4: almost no ratio leaves the clip band.  Here every token row draws one regime, in equal shares: ``plain`` (those
draws), ``shift`` (one constant in [-50, 50] on every logit tensor of the row), ``peaked`` (one logit 25..40 + log V
above the rest; half the rows take it, half take an improbable token), ``flat`` (all logits equal), ``masked`` (the last
5..20 % of V and random columns at -inf or -1e4, never the taken token; some rows have only the taken token finite),
``far`` (``old = new + 3 randn``), ``onpolicy`` (old is new bit for bit), ``large`` (logits x30) and ``kl_far`` (GRPO,
PPO-KL: the reference policy e^20 away).  Independently of the regime, the taken token sits at 0, at V - 1, in the row's
unaligned head or tail, at the edge of the shared-memory row cache or past it, and the row maximum is put in the head or
the tail.  Weights are none, a 0/1 mask with an all-zero sequence, or fractional; advantages include exact zeros and RLOO
rewards with a 1e3 offset and a 1e-2 spread, or K equal rewards.  Shapes sit on both sides of every hand-off of the row
plan: V with no vector at all, one partial vector loop, the unrolled loop and its remainder, exactly the 220 KB row cache
(fp32 V = 56 320, bf16 V = 112 640) and a vector or a few past it, and V = 152 063 / 152 064; row counts 1, 131..133,
529, 4099 and 16 384 around the persistent grid (132 x resident CTAs); sequence lengths 1 and 3 (< grid) and 1500
(>> grid) with weights; token-head sequences of 1, 255..257 and 1100 tokens against its 256 threads, B above its grid.

Reference: ``grpo_oracle.run64`` / ``ppo_lm_oracle.run64`` in float64 on the device.  Yardstick: the same restatements
in float32 on the same inputs (bf16 logits widened to fp32, exactly: DESIGN's contract for bf16 logits).  For every output
X, over the whole tensor and again over the rows of each regime alone,

    max|X_gpu - X_64| <= K * max(max|X_32 - X_64|, 2^-24 * scale_X)

(``test_offpolicy_fp64.compare64``, K = 8).  Loss scales are the fp64 mean of the per-token |term|; a gradient row is
divided by its coefficient scale first (the size of the terms that make up d loss / d lp_new), so that a row with a small
coefficient is not hidden behind a large one.  lse, lp (log-prob methods) and the PPO entropy are checked per row.  A bf16
gradient entry may also differ from the fp64 one by half a bf16 ulp of it (the store's rounding).  Rows whose fp64 ratio
lies within fp32 rounding of fp32(1 -+ clip) or of the dual-clip floor are left out of the elementwise gradient check but
must be finite, and count against compare64's limit.  Every case runs the forward without and with a gradient (uncached
and cached row), the forward-written gradient (unit upstream, skipped on the device), a recompute for a mixed upstream
(0.37, -2, 0 in turn and always nextafter(1, 2), each into a buffer poisoned beforehand) and a repeated backward.  Rows
whose ratio overflows fp32 but not fp64 are a regime of their own: there the GPU must match the fp32 yardstick's
non-finite pattern.  Each case prints its worst ratio to the bound.
"""
import functools
import math
from collections import OrderedDict

import numpy as np
import pytest
import torch

from tests import grpo_oracle as go
from tests import ppo_lm_oracle as po
from tests.test_offpolicy_fp64 import EPS32, K, compare64, policy_terms
from tests.test_value_td_fp64 import _regimes

assert K == 8.0  # the bound of the PPO-family fp64 suite, shared, not loosened here
DEV = 'cuda'
F32, BF16 = torch.float32, torch.bfloat16
REGIMES = ('plain', 'shift', 'peaked', 'flat', 'masked', 'far', 'onpolicy', 'large', 'kl_far')
PLACES = ('rand', 'zero', 'last', 'head', 'tail', 'cache_edge', 'uncached')
CACHE_BYTES = 220 * 1024  # csrc/vocab.cu VOCAB_SMEM_CAP
NEXT1 = float(np.nextafter(np.float32(1), np.float32(2)))
UPSTREAMS = (0.37, -2.0, 0.0)
PPO_MIX = (1.0, -0.01, 0.1)  # the upstream gradients recorded first (forward-written path)
POISON = 7.0


# ----------------------------------------------------------------------------------------------------------------
# the row plan of csrc/vocab.cu, and the generator
# ----------------------------------------------------------------------------------------------------------------
def row_layout(rows, V, esize, chunk=None):
    """per row: the unaligned head length h, the tail start tail0 and the end of the cached part (as vocab_rows_kernel
    splits a row whose byte offset row * V * esize is not a multiple of 16).  ``chunk``: the rows of one chunk buffer of the
    hidden-state losses, whose kernel sees row r at r mod chunk"""
    W = 16 // esize
    r = torch.arange(rows, dtype=torch.int64)
    mis = ((r if chunk is None else r % chunk) * V * esize % 16) // esize
    h = torch.where(mis > 0, torch.clamp(W - mis, max=V), torch.zeros_like(mis))
    tail0 = h + (V - h) // W * W
    capv = min((V * esize + 15) // 16, CACHE_BYTES // 16)
    return h, tail0, torch.minimum(h + capv * W, tail0)


def _pick(u, lo, hi):
    """an index in [lo, hi) from uniform u (rows where hi <= lo give -1)"""
    n = hi - lo
    return torch.where(n > 0, lo + torch.clamp((u * n.clamp(min=1)).long(), max=(n - 1).clamp(min=0)),
                       torch.full_like(lo, -1))


def _placements(g, rows, V, esize, chunk=None):
    """(position class, taken-token position or -1, row-max position class, row-max position or -1)"""
    h, tail0, cend = row_layout(rows, V, esize, chunk)
    u = torch.rand(rows, generator=g)
    zero = torch.zeros(rows, dtype=torch.int64)
    cand = torch.stack([torch.full((rows, ), -1), zero, zero + V - 1, _pick(u, zero, h), _pick(u, tail0, zero + V),
                        torch.where(cend < tail0, cend - 1 + (u < 0.5).long(), -1), _pick(u, cend, tail0)], 1)
    cls = torch.randint(0, len(PLACES), (rows, ), generator=g)
    pos = cand[torch.arange(rows), cls]
    cls = torch.where(pos < 0, torch.zeros_like(cls), cls)
    mcls = torch.randint(0, 4, (rows, ), generator=g)  # 0, 1: nowhere in particular; 2: head; 3: tail
    u2 = torch.rand(rows, generator=g)
    mpos = torch.where(mcls == 2, _pick(u2, zero, h), torch.where(mcls == 3, _pick(u2, tail0, zero + V), -1))
    return cls, pos, torch.where(mpos < 0, torch.zeros_like(mcls), mcls), mpos


def gen_rows(seed, rows, V, dtype, names=REGIMES, with_ref=True, mask_values=(-math.inf, -1e4), chunk=None):
    """rows token rows of V logits: new, old, ref (None without), action and meta (regime per row, placements, masks).
    ``mask_values``: the masked regime's (hard, soft) logit -- a finite hard one where the logits come out of a GEMM, in
    which -inf * 0 is NaN; ``chunk``: place tokens by their row in a chunk buffer of that many rows (row_layout)"""
    g = torch.Generator().manual_seed(seed)
    esize = 4 if dtype == F32 else 2
    reg = _regimes(g, rows, names)
    ri = {nm: reg == i for i, nm in enumerate(names)}
    for nm in REGIMES:
        ri.setdefault(nm, torch.zeros(rows, dtype=torch.bool))
    base = torch.randn(rows, V, generator=g) * 2.0
    n_old = 0.1 * torch.randn(rows, V, generator=g)
    n_ref = 0.2 * torch.randn(rows, V, generator=g)
    action = torch.randint(0, V, (rows, ), generator=g)
    cls, pos, mcls, mpos = _placements(g, rows, V, esize, chunk)
    action = torch.where(pos >= 0, pos, action)
    r = torch.arange(rows)
    has_m = mpos >= 0
    base[r[has_m], mpos[has_m]] = base[has_m].max(1).values + 1.0  # the row max in the head or the tail
    c = torch.rand(rows, 1, generator=g) * 100.0 - 50.0
    new = base.clone()
    new[ri['shift']] += c[ri['shift']]
    # peaked: half the rows take the peak, half an improbable token (the peak elsewhere: the placed max or at random)
    take = torch.rand(rows, generator=g) < 0.5
    other = torch.randint(0, V, (rows, ), generator=g)
    other = torch.where(has_m, mpos, other)
    other = torch.where(other == action, (other + 1) % V, other)
    peak = torch.where(take, action, other)
    pk = ri['peaked'] & (V > 1)
    gap = 25.0 + 15.0 * torch.rand(rows, generator=g) + math.log(max(V, 1))
    new[r[pk], peak[pk]] = base[pk].max(1).values + gap[pk]
    new[ri['flat']] = c[ri['flat']]
    new[ri['large']] *= 30.0
    kf = ri['kl_far']
    new[r[kf], action[kf]] -= 20.0
    old = new + n_old
    old[ri['far']] = new[ri['far']] + 3.0 * torch.randn(int(ri['far'].sum()), V, generator=g)
    old[ri['onpolicy']] = new[ri['onpolicy']]
    old[ri['large']] = new[ri['large']] + 30.0 * n_old[ri['large']]
    c2 = torch.rand(rows, 1, generator=g) * 100.0 - 50.0
    old[ri['flat']] = c2[ri['flat']]
    ref = None
    if with_ref:
        ref = new + n_ref
        ref[ri['large']] = new[ri['large']] + 30.0 * n_ref[ri['large']]
        ref[ri['kl_far']] = base[ri['kl_far']] + n_ref[ri['kl_far']]
        ref[ri['flat']] = (c + c2)[ri['flat']] * 0.5
    # masked: the padded tail of the vocabulary plus random columns; a quarter of the rows keep only the taken token
    mr = ri['masked'] & (V > 1)
    frac = 0.05 + 0.15 * torch.rand(rows, generator=g)
    col = torch.arange(V).unsqueeze(0)
    mask = (col >= (V * (1 - frac)).ceil().long().unsqueeze(1)) | (torch.rand(rows, V, generator=g) < 0.1)
    only = mr & (torch.rand(rows, generator=g) < 0.25)
    mask |= only.unsqueeze(1)
    mask &= mr.unsqueeze(1)
    mask[r, action] = False
    mval = torch.where(only | (torch.rand(rows, generator=g) < 0.5), mask_values[0],
                       mask_values[1]).unsqueeze(1).expand(rows, V)
    for x in (new, old) + ((ref, ) if ref is not None else ()):
        x[mask] = mval[mask]
    out = [x.to(dtype) for x in (new, old)] + [None if ref is None else ref.to(dtype)]
    meta = dict(regime=reg.numpy(), names=tuple(names), place=cls.numpy(), pos=pos.numpy(), mplace=mcls.numpy(),
                mpos=mpos.numpy(), peaked_take=(pk & take).numpy(), only=only.numpy(), mask=mask, esize=esize, chunk=chunk)
    return out[0], out[1], out[2], action, meta


def _weights(g, B, S, wkind, zero_seq=True):
    if wkind is None:
        return None
    if wkind == 'frac':
        return torch.rand(B, S, generator=g)
    w = (torch.rand(B, S, generator=g) > 0.3).float()
    w[:, 0] = 1.0
    if zero_seq and B >= 3:
        w[B // 2] = 0.0  # a sequence without any weight: the reference's loss is NaN (0 / 0), and so must ours be
    return w


def _rewards(g, K, Bp):
    """(K, Bp): a third of the prompts N(0, 1), a third 1e3 + 1e-2 N(0, 1) (cancellation), a third K equal rewards"""
    kind = torch.arange(Bp) % 3
    r = torch.randn(K, Bp, generator=g)
    r = torch.where(kind == 1, 1e3 + 1e-2 * r, r)
    return torch.where(kind == 2, (1e3 + 1e-2 * torch.randn(1, Bp, generator=g)).expand(K, Bp), r)


def a2c_side(g, B, S):
    """(adv, return_, value) (B, S): adv with 10 % exact zeros; returns N(0, 1) or 1e3 + 1e-2 N(0, 1) (cancellation in
    return - value), value == return exactly in a fifth of the tokens"""
    adv = torch.randn(B, S, generator=g)
    adv[torch.rand(B, S, generator=g) < 0.1] = 0.0
    u = torch.rand(B, S, generator=g)
    ret = torch.where(u < 0.4, 1e3 + 1e-2 * torch.randn(B, S, generator=g), torch.randn(B, S, generator=g))
    value = ret + torch.where(ret > 500, 1e-2, 1.0) * torch.randn(B, S, generator=g)
    value = torch.where(torch.rand(B, S, generator=g) < 0.2, ret, value)
    return adv, ret, value


def gen_lm(seed, kind, B, S, V, dtype, wkind, K=0, names=None):
    """grpo / rloo / ppo case dict (CPU) and meta"""
    names = names or (REGIMES if kind in ('grpo', 'ppo_kl') else REGIMES[:-1])
    new, old, ref, action, meta = gen_rows(seed, B * S, V, dtype, names, with_ref=kind in ('grpo', 'ppo_kl'))
    g = torch.Generator().manual_seed(seed + 1)
    d = {'logit_new': new.reshape(B, S, V), 'logit_old': old.reshape(B, S, V), 'action': action.reshape(B, S),
         'weight': _weights(g, B, S, wkind)}
    if kind == 'grpo':
        d['logit_ref'] = ref.reshape(B, S, V)
        d['adv'] = torch.randn(B, generator=g)
        d['adv'][::7] = 0.0
    elif kind == 'rloo':
        d['reward'] = _rewards(g, K, B // K)
    else:
        d['logit_pretrained'] = None if ref is None else ref.reshape(B, S, V)
        adv = torch.randn(B, S, generator=g)
        adv[torch.rand(B, S, generator=g) < 0.05] = 0.0
        d['adv'] = adv
    return d, meta


# ----------------------------------------------------------------------------------------------------------------
# per-token terms in float64: boundary rows, loss scales, gradient-row scales
# ----------------------------------------------------------------------------------------------------------------
def _lp64(x, a):
    x = x.double()
    return (x.gather(-1, a.unsqueeze(-1)).squeeze(-1) - torch.logsumexp(x, -1)).reshape(-1).cpu().numpy()


def _boundary(ratio, adv, lse_sz, dual_clip=None, clip=go.CLIP):
    """rows whose fp64 ratio lies within fp32 rounding of a clamp bound (or of the dual-clip floor, adv < 0): the fp32 log
    ratio carries a few ulps of the logsumexps and logits it is made of"""
    lr = np.log(np.maximum(ratio, 1e-300))
    win = 4 * EPS32 * (1.0 + lse_sz)
    bounds = [float(np.float32(1 - clip)), float(np.float32(1 + clip))]
    bnd = np.zeros(ratio.shape, bool)
    for b in bounds:
        bnd |= np.abs(lr - math.log(b)) <= win
    if dual_clip:
        bnd |= (adv < 0) & (np.abs(lr - math.log(dual_clip)) <= win)
    return bnd


def _lse_size(d, keys):
    """per row: sum of |logsumexp| and |taken logit| over the logit tensors (what an fp32 log ratio is rounded against)"""
    tot = 0.0
    for k in keys:
        x = d[k].double()
        lse = torch.logsumexp(x, -1).abs()
        za = x.gather(-1, d['action'].unsqueeze(-1)).squeeze(-1).abs()
        tot = tot + (lse + torch.nan_to_num(za, posinf=0.0)).reshape(-1).cpu().numpy()
    return tot


def grpo_meta(kind, d):
    """(boundary rows, loss scales) of a grpo / rloo case"""
    a = d['action']
    lpn, lpo = _lp64(d['logit_new'], a), _lp64(d['logit_old'], a)
    B, S = a.shape
    adv = (d['adv'].double().cpu() if kind == 'grpo' else go.rloo_adv64(d['reward'].cpu())).numpy()
    adv_r = np.repeat(adv, S)
    ratio = np.exp(lpn - lpo)
    w = np.ones((B, S)) if d['weight'] is None else d['weight'].double().cpu().numpy()
    with np.errstate(invalid='ignore', divide='ignore'):
        wn = (w / w.sum(1, keepdims=True)).reshape(-1)
    rc = np.clip(ratio, 1 - go.CLIP, 1 + go.CLIP)
    tok = np.abs(np.minimum(ratio * adv_r, rc * adv_r))
    if kind == 'grpo':
        dr = _lp64(d['logit_ref'], a) - lpn
        tok = tok + go.BETA * np.abs(np.exp(dr) - dr - 1)
    keys = ('logit_new', 'logit_old')
    bnd = _boundary(ratio, adv_r, _lse_size(d, keys))
    scales = {'out_loss': float(np.nansum(tok * wn)) / B, 'out_approx_kl': float(np.mean(np.abs(lpo - lpn)))}
    return bnd, scales


def ppo_meta(d, p, mix):
    """(boundary rows, loss scales, per-row gradient scale for the upstream mix) of a PPO-LM case"""
    a = d['action']
    lpn, lpo = _lp64(d['logit_new'], a), _lp64(d['logit_old'], a)
    ratio = np.exp(lpn - lpo)
    adv = d['adv'].double().reshape(-1).cpu().numpy()
    M = adv.size
    w = np.ones(M) if d['weight'] is None else d['weight'].double().reshape(-1).cpu().numpy()
    _, _, pol = policy_terms(ratio, adv, w, np.ones(M), go.CLIP, p['dual_clip'])
    bnd = _boundary(ratio, adv, _lse_size(d, ('logit_new', 'logit_old')), p['dual_clip'])
    scales = {'out_policy': pol, 'out_approx_kl': float(np.mean(np.abs(lpo - lpn)))}
    row = np.abs(mix[0]) * w * np.abs(adv) * ratio
    if p['entropy_bonus']:
        x = d['logit_new'].double()
        lsm = torch.log_softmax(x, -1)
        H = -(torch.exp(lsm) * lsm.clamp(min=torch.finfo(torch.float64).min)).sum(-1).reshape(-1).cpu().numpy()
        scales['out_entropy'] = float(np.mean(np.abs(H * w)))
        row = row + np.abs(mix[1]) * w * (1.0 + H)
    if d['logit_pretrained'] is not None:
        lr = lpn - _lp64(d['logit_pretrained'], a)
        kt = {'k1': lr, 'k2': lr ** 2 / 2, 'k3': np.exp(-lr) - 1 + lr}[p['kl_type']]
        scales['out_kl'] = float(np.mean(np.abs(kt)))
        row = row + np.abs(mix[2]) * (1.0 + np.abs(lr) + np.exp(-lr))
    return bnd, scales, row / M


# ----------------------------------------------------------------------------------------------------------------
# the comparison: whole tensor, then each regime's rows alone
# ----------------------------------------------------------------------------------------------------------------
def bf16_rounding(x, b):
    """x moved towards b by up to half a bf16 ulp of b: the rounding of the kernel's fp32 value to a bf16 gradient"""
    with np.errstate(divide='ignore', invalid='ignore'):
        e = np.floor(np.log2(np.abs(b)))
        hu = np.where(np.isfinite(e), np.exp2(e - 8), 0.0)
        dd = x - b
        out = b + np.sign(dd) * np.maximum(np.abs(dd) - hu, 0.0)
    return np.where(np.isfinite(x) & np.isfinite(b), out, x)


def row_divisor(scale):
    s = np.asarray(scale, np.float64).reshape(-1)
    return np.where(np.isfinite(s) & (s > 0), s, 1.0)


def compare_regimes(tag, got, r32, r64, meta, scales=None, bnd=None):
    """compare64 over the whole tensors, then over the rows of each regime (the per-row outputs: lse, lp, ent, grad_*);
    returns the worst ratio"""
    n = len(meta['regime'])
    worst = compare64(tag, got, r32, r64, scales=scales, bnd=bnd, S=n)
    keys = [k for k in r64 if np.ndim(r64[k]) >= 1 and np.shape(r64[k])[0] == n]
    for i, nm in enumerate(meta['names']):
        m = meta['regime'] == i
        if not m.any() or m.all() or not keys:
            continue
        sub = [OrderedDict((k, np.asarray(dd[k])[m]) for k in keys) for dd in (got, r32, r64)]
        w = compare64('%s [%s]' % (tag, nm), *sub, bnd=None if bnd is None else bnd[m])
        worst = max(worst, w)
        WORST.setdefault(nm, [0.0, ''])
        if w > WORST[nm][0]:
            WORST[nm] = [w, tag]
    return worst


WORST = {}  # regime -> [worst ratio, path] of the running case: cleared when a case starts, printed when it ends


def _per_regime():
    return {k: round(v[0], 2) for k, v in WORST.items()}


def grad_entry(x, div, bf16, want64=None):
    """(rows, V) float64 numpy gradient divided row by row by its scale; a bf16 gradient first loses the store's
    rounding against the fp64 one"""
    x = x.detach().double().reshape(len(div), -1).cpu().numpy()
    if bf16 and want64 is not None:
        x = bf16_rounding(x, want64)
    return x / div[:, None]


def _np(x):
    return x.detach().double().cpu().numpy() if torch.is_tensor(x) else np.float64(x)


# ----------------------------------------------------------------------------------------------------------------
# GRPO / RLOO through the fused launch
# ----------------------------------------------------------------------------------------------------------------
GR_CASES = {
    # name: (kind, dtype, B, S, V, weight kind, K)
    'grpo_f32_v1_r16384': ('grpo', F32, 16, 1024, 1, 'frac', 0),
    'grpo_f32_v3_r529': ('grpo', F32, 23, 23, 3, None, 0),
    'grpo_f32_v1027_s1500': ('grpo', F32, 3, 1500, 1027, 'frac', 0),
    'grpo_f32_v1027_r4099_s1': ('grpo', F32, 4099, 1, 1027, 'frac', 0),
    'grpo_f32_v2048_r133_zero_seq': ('grpo', F32, 7, 19, 2048, 'mask', 0),
    'grpo_f32_v4100_r529': ('grpo', F32, 23, 23, 4100, None, 0),
    'grpo_f32_v56320_r131': ('grpo', F32, 131, 1, 56320, 'frac', 0),
    'grpo_f32_v56324_r133': ('grpo', F32, 1, 133, 56324, None, 0),
    'grpo_f32_v56333_r132_s3': ('grpo', F32, 44, 3, 56333, 'frac', 0),
    'grpo_f32_v152063_r3': ('grpo', F32, 1, 3, 152063, 'frac', 0),
    'grpo_bf16_v1_r1': ('grpo', BF16, 1, 1, 1, None, 0),
    'grpo_bf16_v7_r16384_zero_seq': ('grpo', BF16, 16, 1024, 7, 'mask', 0),
    'grpo_bf16_v9_r529': ('grpo', BF16, 23, 23, 9, 'frac', 0),
    'grpo_bf16_v1003_s1500': ('grpo', BF16, 2, 1500, 1003, 'frac', 0),
    'grpo_bf16_v4096_r529': ('grpo', BF16, 23, 23, 4096, None, 0),
    'grpo_bf16_v8200_r133_zero_seq': ('grpo', BF16, 7, 19, 8200, 'mask', 0),
    'grpo_bf16_v112640_r131': ('grpo', BF16, 131, 1, 112640, 'frac', 0),
    'grpo_bf16_v112648_r133': ('grpo', BF16, 1, 133, 112648, None, 0),
    'grpo_bf16_v112647_r132_s3': ('grpo', BF16, 44, 3, 112647, 'frac', 0),
    'grpo_bf16_v152064_r3': ('grpo', BF16, 3, 1, 152064, None, 0),
    'rloo_f32_k2_v1027_r532': ('rloo', F32, 4, 133, 1027, 'frac', 2),
    'rloo_f32_k3_v4100_r132': ('rloo', F32, 6, 22, 4100, 'mask', 3),
    'rloo_f32_k64_v3_r512': ('rloo', F32, 128, 4, 3, None, 64),
    'rloo_bf16_k8_v8200_r144': ('rloo', BF16, 16, 9, 8200, 'mask', 8),
    'rloo_bf16_k64_v9_r4099': ('rloo', BF16, 4096, 1, 9, 'frac', 64),
    'rloo_bf16_k2_v112648_r4': ('rloo', BF16, 2, 2, 112648, None, 2),
}


def _to(d, dev):
    return {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in d.items()}


@functools.lru_cache(maxsize=1)
def _gr_case(name):
    kind, dtype, B, S, V, wkind, Kr = GR_CASES[name]
    d, meta = gen_lm(9300 + list(GR_CASES).index(name), kind, B, S, V, dtype, wkind, Kr)
    d = _to(d, DEV)
    bnd, scales = grpo_meta(kind, d)
    rr = {}
    for dt in (torch.float64, torch.float32):
        r = go.run64(d, dtype=dt)
        grad = torch.stack([go.grad_rows64(d['logit_new'][b], d['action'][b], r['dlp'][b], dt) for b in range(B)])
        rr[dt] = dict(r, grad=grad.reshape(B * S, V), lse=torch.logsumexp(d['logit_new'].to(dt), -1).reshape(-1))
    div = row_divisor(rr[torch.float64]['scale'].cpu().numpy())
    return kind, d, meta, bnd, scales, rr, div


def _gr_refs(rr, div, g, with_grad):
    out = []
    for dt in (torch.float32, torch.float64):
        r = rr[dt]
        res = OrderedDict([('out_loss', r['loss']),
                           ('out_approx_kl', r['approx_kl']), ('out_clipfrac', r['clipfrac'])])
        if with_grad:
            res['lse'] = _np(r['lse'])
            gr = r['grad'] * torch.tensor(g, dtype=dt) if g != 1.0 else r['grad']
            res['grad_logit_new'] = _np(gr) / div[:, None]
        out.append(res)
    return out


def _gr_call(kind, d, x):
    import di_engine_b200 as b2
    R = b2.rl_utils
    if kind == 'grpo':
        return R.grpo_policy_error(R.grpo_policy_data(x, d['logit_old'], d['logit_ref'], d['action'], d['adv'],
                                                      d['weight']))
    return R.rloo_policy_error(R.rloo_policy_data(x, d['logit_old'], d['action'], d['reward'], d['weight']))


def _gr_run(kind, d, div, bf16, want64, grad, g=1.0, poison=False, twice=False):
    x = d['logit_new'].clone().requires_grad_(grad)
    loss, info = _gr_call(kind, d, x)
    res = OrderedDict([('out_loss', loss.item()), ('out_approx_kl', info.approx_kl), ('out_clipfrac', info.clipfrac)])
    if not grad:
        return res
    fn = loss.grad_fn
    res['lse'] = _np(fn.saved_tensors[2])
    if poison:
        fn.spec.fill_(POISON)  # a recompute overwrites every entry; a skipped launch would leave this
    (loss * g if g != 1.0 else loss).backward(retain_graph=twice)
    if twice:
        loss.backward()
    res['grad_logit_new'] = grad_entry(x.grad, div, bf16, want64)
    return res


@pytest.mark.gpu
@pytest.mark.parametrize('name', list(GR_CASES))
def test_grpo_rloo_fp64(name):
    kind, d, meta, bnd, scales, rr, div = _gr_case(name)
    bf16 = d['logit_new'].dtype == BF16
    want64 = _np(rr[torch.float64]['grad'])
    worst = 0.0
    WORST.clear()
    # the forward alone (no gradient, no row cache)
    r32, r64 = _gr_refs(rr, div, 1.0, False)
    worst = max(worst, compare_regimes(name + ' nograd', _gr_run(kind, d, div, bf16, None, False), r32, r64, meta,
                                       scales, bnd))
    g_mixed = UPSTREAMS[list(GR_CASES).index(name) % len(UPSTREAMS)]
    for path, g, poison, twice in (('unit', 1.0, False, False), ('next1', NEXT1, True, False),
                                   ('mixed %g' % g_mixed, g_mixed, True, False), ('twice', 2.0, False, True)):
        got = _gr_run(kind, d, div, bf16, want64 * (g if path != 'twice' else 2.0), True,
                      g if path != 'twice' else 1.0, poison, twice)
        r32, r64 = _gr_refs(rr, div, g, True)
        worst = max(worst, compare_regimes('%s %s' % (name, path), got, r32, r64, meta, scales, bnd))
    print('[fp64] %s worst %.2f  per regime %s' % (name, worst, _per_regime()))


# ----------------------------------------------------------------------------------------------------------------
# PPO on token rows: entropy x KL x dual clip, fp32 (V >= 1024) and bf16
# ----------------------------------------------------------------------------------------------------------------
def _ppo_grid():
    out = OrderedDict()
    i = 0
    for dtype, V in ((F32, 1027), (BF16, 1003)):
        for ent in (False, True):
            for kl in (None, 'k1', 'k2', 'k3'):
                for dc in (None, 2.0):
                    wk = (None, 'mask', 'frac')[i % 3]
                    out['ppo_%s_v%d_%s_%s_%s' % ('f32' if dtype == F32 else 'bf16', V, 'ent' if ent else 'noent',
                                               kl or 'nokl', 'dc' if dc else 'nodc')] = (dtype, 23, 23, V, wk, ent,
                                                                                         kl, dc)
                    i += 1
    out['ppo_f32_v56324_r133_ent_k3_dc'] = (F32, 7, 19, 56324, 'frac', True, 'k3', 2.0)
    out['ppo_f32_v4100_r4099_ent_k2'] = (F32, 4099, 1, 4100, 'mask', True, 'k2', None)
    out['ppo_bf16_v112647_r133_ent_k1_dc'] = (BF16, 1, 133, 112647, None, True, 'k1', 2.0)
    out['ppo_bf16_v152064_r3_ent_k3'] = (BF16, 1, 3, 152064, 'frac', True, 'k3', None)
    return out


PPO_CASES = _ppo_grid()
PPO_MIXES = (PPO_MIX, (NEXT1, -0.01, 0.1), (0.37, -2.0, 0.0), (-2.0, 0.37, 0.37), (0.0, 0.0, 0.0))


@functools.lru_cache(maxsize=1)
def _ppo_case(name):
    dtype, B, S, V, wk, ent, kl, dc = PPO_CASES[name]
    d, meta = gen_lm(9500 + list(PPO_CASES).index(name), 'ppo_kl' if kl else 'ppo', B, S, V, dtype, wk)
    d = _to(d, DEV)
    p = dict(dual_clip=dc, kl_type=kl or 'k1', entropy_bonus=ent)
    parts = {}
    for dt in (torch.float64, torch.float32):
        res = []
        for unit in ((1.0, 0.0, 0.0), (0.0, 1.0, 0.0), (0.0, 0.0, 1.0)):
            res.append(po.run64(d, dual_clip=dc, kl_type=p['kl_type'], entropy_bonus=ent, mix=unit, dtype=dt))
        parts[dt] = res
    return d, meta, p, parts


def _ppo_refs(d, p, parts, mix, div, scale_mult=1.0):
    out = []
    for dt in (torch.float32, torch.float64):
        r = parts[dt]
        res = OrderedDict([('out_policy', r[0]['policy']), ('out_entropy', r[0]['entropy']), ('out_kl', r[0]['kl']),
                           ('out_approx_kl', r[0]['approx_kl']), ('out_clipfrac', r[0]['clipfrac'])])
        res['lse'] = _np(r[0]['lse'].reshape(-1))
        if p['entropy_bonus']:
            res['ent'] = _np(r[0]['H'].reshape(-1))
        gr = sum(torch.tensor(m * scale_mult, dtype=dt, device=r[0]['grad'].device) * ri['grad']
                 for m, ri in zip(mix, r))
        res['grad_logit_new'] = _np(gr.reshape(div.size, -1)) / div[:, None]
        out.append(res)
    return out


def _ppo_run(d, p, mix, div, bf16, want64, poison=False, twice=False, grad=True):
    import di_engine_b200 as b2
    R = b2.rl_utils
    x = d['logit_new'].clone().requires_grad_(grad)
    loss, info = R.ppo_policy_error(R.ppo_policy_data(x, d['logit_old'], d['action'], d['adv'], d['weight'],
                                                      d['logit_pretrained']), clip_ratio=po.CLIP, **p)
    res = OrderedDict([('out_policy', loss.policy_loss.item()), ('out_entropy', float(loss.entropy_loss)),
                       ('out_kl', loss.kl_div.item()), ('out_approx_kl', info.approx_kl),
                       ('out_clipfrac', info.clipfrac)])
    if not grad:
        return res
    fn = loss.policy_loss.grad_fn
    saved = fn.saved_tensors
    res['lse'] = _np(saved[3])
    if p['entropy_bonus']:
        res['ent'] = _np(saved[4])
    if poison:
        fn.spec[0].fill_(POISON)
    total = mix[0] * loss.policy_loss
    if p['entropy_bonus']:
        total = total + mix[1] * loss.entropy_loss
    if d['logit_pretrained'] is not None:
        total = total + mix[2] * loss.kl_div
    total.backward(retain_graph=twice)
    if twice:
        total.backward()
    res['grad_logit_new'] = grad_entry(x.grad, div, bf16, want64)
    return res


@pytest.mark.gpu
@pytest.mark.parametrize('name', list(PPO_CASES))
def test_ppo_lm_fp64(name):
    from di_engine_b200 import ops
    d, meta, p, parts = _ppo_case(name)
    bf16 = d['logit_new'].dtype == BF16
    hint = ops.ppo_hint(torch.device(DEV, torch.cuda.current_device()), 'policy')  # the record the calls read
    saved_hint = hint.clone()
    worst = 0.0
    WORST.clear()
    try:
        bnd, scales, _ = ppo_meta(d, p, PPO_MIX)
        got = _ppo_run(d, p, PPO_MIX, np.ones(len(meta['regime'])), bf16, None, grad=False)
        r32, r64 = _ppo_refs(d, p, parts, PPO_MIX, np.ones(len(meta['regime'])))
        for dd in (r32, r64):
            dd.pop('lse'), dd.pop('ent', None), dd.pop('grad_logit_new')
        worst = compare_regimes(name + ' nograd', got, r32, r64, meta, scales, bnd)
        hint.copy_(torch.tensor([PPO_MIX[0], 0.0, PPO_MIX[1], PPO_MIX[2]]))  # the first step records the mix
        paths = [('expected', PPO_MIX, False, False)] + [('mix %s' % (m, ), m, True, False) for m in PPO_MIXES[1:]]
        paths.append(('twice', PPO_MIX, False, True))
        for path, mix, poison, twice in paths:
            mult = 2.0 if twice else 1.0
            _, _, row = ppo_meta(d, p, mix)
            div = row_divisor(row * mult)
            r32, r64 = _ppo_refs(d, p, parts, mix, div, mult)
            got = _ppo_run(d, p, mix, div, bf16, r64['grad_logit_new'] * div[:, None], poison, twice)
            worst = max(worst, compare_regimes('%s %s' % (name, path), got, r32, r64, meta, scales, bnd))
    finally:
        hint.copy_(saved_hint)
    print('[fp64] %s worst %.2f  per regime %s' % (name, worst, _per_regime()))


# ----------------------------------------------------------------------------------------------------------------
# the log-prob methods (LogpRow, CoefBwdRow with a per-row upstream)
# ----------------------------------------------------------------------------------------------------------------
LP_CASES = OrderedDict(
    [('f32_v%d_r%d' % (V, r), (F32, r, V)) for V, r in ((1, 16384), (3, 4099), (1027, 529), (2048, 133), (4100, 132),
                                                         (56320, 131), (56324, 133), (56333, 133), (152063, 7))] +
    [('bf16_v%d_r%d' % (V, r), (BF16, r, V)) for V, r in ((1, 1), (7, 16384), (9, 529), (1003, 4099), (4096, 133),
                                                          (8200, 132), (112640, 131), (112648, 133), (112647, 67),
                                                          (152064, 7))])
LP_METHODS = ('naive_method', 'efficient_method', 'less_efficient_method')


@pytest.mark.gpu
@pytest.mark.parametrize('name', list(LP_CASES))
def test_log_prob_fp64(name):
    import di_engine_b200 as b2
    dtype, rows, V = LP_CASES[name]
    new, _, _, action, meta = gen_rows(9700 + list(LP_CASES).index(name), rows, V, dtype, REGIMES[:-1], False)
    x0, a = new.to(DEV), action.to(DEV)
    g = torch.Generator().manual_seed(9800 + rows)
    up = torch.randn(rows, generator=g)
    up[torch.rand(rows, generator=g) < 0.1] = 0.0
    up[:4] = torch.tensor([0.37, -2.0, 0.0, NEXT1])[:rows]
    up = up.to(DEV)
    div = row_divisor(up.abs().cpu().numpy())
    refs = []
    for dt in (torch.float32, torch.float64):
        lp = go.logp64(x0, a, dt)
        gr = go.grad_rows64(x0, a, up.to(dt), dt)
        refs.append(OrderedDict([('lp', _np(lp)), ('grad_logits', _np(gr) / div[:, None])]))
    want64 = _np(go.grad_rows64(x0, a, up.double()))
    worst = 0.0
    WORST.clear()
    methods = LP_METHODS if list(LP_CASES).index(name) % 4 == 0 else LP_METHODS[1:2]
    for m in methods:
        for shape in ((rows, V), (1, rows, V)):
            x = x0.reshape(shape).clone().requires_grad_(True)
            lp = getattr(b2.rl_utils, m)(x, a.reshape(shape[:-1]))
            (lp * up.reshape(shape[:-1])).sum().backward()
            got = OrderedDict([('lp', _np(lp.reshape(-1))), ('grad_logits', grad_entry(x.grad, div, dtype == BF16,
                                                                                        want64))])
            worst = max(worst, compare_regimes('logp %s %s %s' % (name, m, shape), got, *refs, meta))
    print('[fp64] logp %s worst %.2f  per regime %s' % (name, worst, _per_regime()))


# ----------------------------------------------------------------------------------------------------------------
# the token head on a custom log_prob_fn's output (token_head_kernel)
# ----------------------------------------------------------------------------------------------------------------
HEAD_B = 1100  # above the head kernel's grid (132 SMs x its resident CTAs of 256 threads)


def _head_lps(seed, B, S):
    """per-token (lp_new, lp_old, lp_ref) drawn as log-probabilities of the regimes: near 0 (peaked, taken), about -35
    (improbable), on-policy, far, kl_far"""
    g = torch.Generator().manual_seed(seed)
    n = B * S
    reg = _regimes(g, n, ('plain', 'peaked', 'far', 'onpolicy', 'kl_far'))
    lpn = -torch.rand(n, generator=g) * 5.0
    pk = reg == 1
    lpn[pk] = torch.where(torch.rand(n, generator=g) < 0.5, -1e-11 * torch.rand(n, generator=g) - 1e-12,
                          -35.0 - torch.rand(n, generator=g))[pk]
    kf = reg == 4
    lpr = (lpn + 0.2 * torch.randn(n, generator=g)).clamp(max=0.0)
    lpn[kf] = lpr[kf] - 20.0 - torch.rand(n, generator=g)[kf]
    lpo = (lpn + 0.1 * torch.randn(n, generator=g)).clamp(max=0.0)
    lpo[reg == 2] = (lpn - 3.0 * torch.randn(n, generator=g)).clamp(max=0.0)[reg == 2]
    lpo[reg == 3] = lpn[reg == 3]
    return [t.reshape(B, S) for t in (lpn, lpo, lpr)], dict(regime=reg.numpy(), names=('plain', 'peaked', 'far',
                                                                                       'onpolicy', 'kl_far'))


@pytest.mark.gpu
@pytest.mark.parametrize('kind', ['grpo', 'rloo'])
@pytest.mark.parametrize('S', [1, 255, 256, 257, 1100])
def test_token_head_fp64(S, kind):
    import di_engine_b200 as b2
    R = b2.rl_utils
    B = HEAD_B if S < 1100 else 1104
    seed = 9900 + S + (kind == 'rloo')
    (lpn, lpo, lpr), meta = _head_lps(seed, B, S)
    g = torch.Generator().manual_seed(seed + 1)
    # 0/1 masks at odd S (an all-zero sequence, whose NaN loss the kernel must give too, only at S = 1), fractional at even
    weight = _weights(g, B, S, 'mask' if S % 2 else 'frac', zero_seq=S == 1)
    side = torch.randn(B, generator=g) if kind == 'grpo' else _rewards(g, 4, B // 4)
    if kind == 'grpo':
        side[::5] = 0.0
    ident = lambda x, a: x  # noqa: E731
    lp_ref = lpr if kind == 'grpo' else None
    beta = go.BETA if kind == 'grpo' else 0.0
    adv64 = side.double() if kind == 'grpo' else go.rloo_adv64(side)
    adv32 = side if kind == 'grpo' else go.rloo_adv64(side, torch.float32)
    refs = []
    for dt, adv in ((torch.float32, adv32), (torch.float64, adv64)):
        x = lpn.to(dt).clone().requires_grad_(True)
        loss, kl, cf = go.head64(x, lpo.to(dt), None if lp_ref is None else lp_ref.to(dt), adv, weight, go.CLIP, beta)
        loss.backward()
        refs.append(OrderedDict([('out_loss', loss.item()), ('out_approx_kl', kl.item()), ('out_clipfrac', cf.item()),
                                 ('grad_lp', x.grad.reshape(-1).double().numpy())]))
    # row scale of the gradient: w / (B sum_s w) * (|adv| ratio [+ beta (exp(lp_ref - lp_new) + 1)])
    w = torch.ones(B, S, dtype=torch.float64) if weight is None else weight.double()
    gt = w / w.sum(1, keepdim=True) / B
    sc = gt * adv64.abs().reshape(-1, 1) * torch.exp(lpn.double() - lpo.double())
    if lp_ref is not None:
        sc = sc + gt * beta * (torch.exp(lpr.double() - lpn.double()) + 1)
    div = row_divisor(sc.reshape(-1).numpy())
    for r in refs:
        r['grad_lp'] = r['grad_lp'] / div
    ratio = np.exp(lpn.double().reshape(-1).numpy() - lpo.double().reshape(-1).numpy())
    bnd = _boundary(ratio, np.repeat(adv64.numpy(), S), np.abs(lpn.double().numpy()).reshape(-1) +
                    np.abs(lpo.double().numpy()).reshape(-1))
    adv_r = np.repeat(adv64.numpy(), S)
    tok = np.abs(np.minimum(ratio * adv_r, np.clip(ratio, 1 - go.CLIP, 1 + go.CLIP) * adv_r))
    if lp_ref is not None:  # the loss scale includes the KL term, as grpo_meta's
        dr = lpr.double().reshape(-1).numpy() - lpn.double().reshape(-1).numpy()
        tok = tok + beta * np.abs(np.exp(dr) - dr - 1)
    with np.errstate(invalid='ignore'):
        scales = {'out_loss': float(np.nansum(tok * (w / w.sum(1, keepdim=True)).reshape(-1).numpy())) / B,
                  'out_approx_kl': float(np.mean(np.abs(lpo.double().numpy() - lpn.double().numpy())))}
    dev = {k: (None if v is None else v.to(DEV)) for k, v in (('lpo', lpo), ('lpr', lp_ref), ('w', weight),
                                                                ('side', side))}
    x = lpn.to(DEV).clone().requires_grad_(True)
    act = torch.zeros(B, S, dtype=torch.long, device=DEV)
    if kind == 'grpo':
        loss, info = R.grpo_policy_error(R.grpo_policy_data(x, dev['lpo'], dev['lpr'], act, dev['side'], dev['w']), ident)
    else:
        loss, info = R.rloo_policy_error(R.rloo_policy_data(x, dev['lpo'], act, dev['side'], dev['w']), ident)
    loss.backward()
    got = OrderedDict([('out_loss', loss.item()), ('out_approx_kl', info.approx_kl), ('out_clipfrac', info.clipfrac),
                       ('grad_lp', x.grad.reshape(-1).double().cpu().numpy() / div)])
    WORST.clear()
    worst = compare_regimes('head %s S=%d' % (kind, S), got, *refs, meta, scales, bnd)
    print('[fp64] head %s S=%d worst %.2f  per regime %s' % (kind, S, worst, _per_regime()))


# ----------------------------------------------------------------------------------------------------------------
# A2C on token rows (A2cRow, backward PgBwdRow with the value slot) and its upstream-gradient record
# ----------------------------------------------------------------------------------------------------------------
A2C_NAMES = ('plain', 'shift', 'peaked', 'flat', 'masked', 'large')  # the regimes without an old policy
A2C_CASES = {
    # name: (dtype, B, S, V, weight kind)
    'a2c_f32_v1_r16384': (F32, 16, 1024, 1, 'frac'),
    'a2c_f32_v3_r529': (F32, 23, 23, 3, None),
    'a2c_f32_v1027_s1500': (F32, 3, 1500, 1027, 'mask'),
    'a2c_f32_v1027_r4099_s1': (F32, 4099, 1, 1027, 'frac'),
    'a2c_f32_v4100_r529': (F32, 23, 23, 4100, None),
    'a2c_f32_v56320_r131': (F32, 131, 1, 56320, 'frac'),
    'a2c_f32_v56324_r133': (F32, 1, 133, 56324, None),
    'a2c_f32_v56333_r132_s3': (F32, 44, 3, 56333, 'mask'),
    'a2c_f32_v152063_r3': (F32, 1, 3, 152063, 'frac'),
    'a2c_bf16_v1_r1': (BF16, 1, 1, 1, None),
    'a2c_bf16_v7_r4099': (BF16, 4099, 1, 7, 'mask'),
    'a2c_bf16_v1003_r529': (BF16, 23, 23, 1003, 'frac'),
    'a2c_bf16_v8200_r133': (BF16, 7, 19, 8200, 'mask'),
    'a2c_bf16_v112640_r131': (BF16, 131, 1, 112640, 'frac'),
    'a2c_bf16_v112648_r133': (BF16, 1, 133, 112648, None),
    'a2c_bf16_v112647_r132_s3': (BF16, 44, 3, 112647, 'frac'),
    'a2c_bf16_v152064_r3': (BF16, 3, 1, 152064, 'frac'),
}
A2C_RECORD = (1.0, 0.5, -0.01)  # ops._HINT_INIT['a2c']: the upstream gradients the forward writes for
# the record; nextafter(1, 2) in the policy slot; the record but for the value slot; (0.37, -2, 0); all zeros
A2C_MIXES = (A2C_RECORD, (NEXT1, 0.5, -0.01), (1.0, 0.37, -0.01), (0.37, -2.0, 0.0), (0.0, 0.0, 0.0))


@functools.lru_cache(maxsize=1)
def _a2c_case(name):
    from oracle import rl_oracle
    dtype, B, S, V, wk = A2C_CASES[name]
    seed = 10100 + list(A2C_CASES).index(name)
    new, _, _, action, meta = gen_rows(seed, B * S, V, dtype, A2C_NAMES, False)
    g = torch.Generator().manual_seed(seed + 1)
    adv, ret, value = a2c_side(g, B, S)
    d = _to({'logit': new.reshape(B, S, V), 'action': action.reshape(B, S), 'weight': _weights(g, B, S, wk),
             'adv': adv, 'return_': ret, 'value': value}, DEV)
    parts = {}
    for dt in (torch.float64, torch.float32):
        res = []
        for unit in ((1.0, 0.0, 0.0), (0.0, 1.0, 0.0), (0.0, 0.0, 1.0)):
            x = d['logit'].to(dt, copy=True).requires_grad_(True)
            v = d['value'].to(dt, copy=True).requires_grad_(True)
            w = None if d['weight'] is None else d['weight'].to(dt)
            p, vl, e = rl_oracle.a2c_error(x, d['action'], v, d['adv'].to(dt), d['return_'].to(dt), w)
            (unit[0] * p + unit[1] * vl + unit[2] * e).backward()
            res.append(dict(policy=p.item(), value=vl.item(), entropy=e.item(), grad=x.grad.reshape(B * S, V),
                            grad_value=v.grad.reshape(-1)))
        parts[dt] = res
    x = d['logit'].double()
    lsm = torch.log_softmax(x, -1)
    H = -(torch.exp(lsm) * lsm.clamp(min=torch.finfo(torch.float64).min)).sum(-1).reshape(-1).cpu().numpy()
    w = np.ones(B * S) if d['weight'] is None else d['weight'].double().reshape(-1).cpu().numpy()
    lp = _lp64(x, d['action'])
    a_ = d['adv'].double().reshape(-1).cpu().numpy()
    dv = (d['return_'] - d['value']).double().reshape(-1).cpu().numpy()
    scales = {'out_policy': float(np.mean(np.abs(lp * a_ * w))), 'out_value': float(np.mean(dv ** 2 * w)),
              'out_entropy': float(np.mean(np.abs(H * w)))}
    return d, meta, parts, scales, (w * np.abs(a_), w * (1.0 + H), w * np.abs(dv))


def _a2c_refs(parts, mix, div, mult=1.0):
    out = []
    for dt in (torch.float32, torch.float64):
        r = parts[dt]
        res = OrderedDict([('out_policy', r[0]['policy']), ('out_value', r[0]['value']),
                           ('out_entropy', r[0]['entropy'])])
        dev = r[0]['grad'].device
        gr = sum(torch.tensor(m * mult, dtype=dt, device=dev) * ri['grad'] for m, ri in zip(mix, r))
        gv = sum(torch.tensor(m * mult, dtype=dt, device=dev) * ri['grad_value'] for m, ri in zip(mix, r))
        res['grad_logit'] = _np(gr) / div[:, None]
        res['grad_value'] = _np(gv)
        out.append(res)
    return out


def _a2c_run(d, mix, div, bf16, want64, poison=False, twice=False, grad=True):
    import di_engine_b200 as b2
    R = b2.rl_utils
    x = d['logit'].clone().requires_grad_(grad)
    v = d['value'].clone().requires_grad_(grad)
    loss = R.a2c_error(R.a2c_data(x, d['action'], v, d['adv'], d['return_'], d['weight']))
    res = OrderedDict([('out_policy', loss.policy_loss.item()), ('out_value', loss.value_loss.item()),
                       ('out_entropy', loss.entropy_loss.item())])
    if not grad:
        return res, None, None
    if poison:
        spec = loss.policy_loss.grad_fn.spec
        spec[0].fill_(POISON)
        spec[1].fill_(POISON)
    total = mix[0] * loss.policy_loss + mix[1] * loss.value_loss + mix[2] * loss.entropy_loss
    total.backward(retain_graph=twice)
    if twice:
        total.backward()
    res['grad_logit'] = grad_entry(x.grad, div, bf16, want64)
    res['grad_value'] = _np(v.grad).reshape(-1)
    return res, x.grad, v.grad


def _bits(a, b):
    return np.float32(a).view(np.uint32) == np.float32(b).view(np.uint32)


@pytest.mark.gpu
@pytest.mark.parametrize('name', list(A2C_CASES))
def test_a2c_lm_fp64(name, monkeypatch):
    """the forward alone, then each mix with the forward's gradient buffers poisoned (the record's policy and entropy
    slots kept: d logit is the forward's, untouched; the value slot too: both), again unpoisoned, and a repeated
    backward (the recompute path); every run starts from the record"""
    import di_engine_b200 as b2
    from di_engine_b200 import ops
    monkeypatch.setattr(b2.rl_utils.ppo, 'LM_MIN_VOCAB', 1)  # fp32 V < 1024 takes the vocabulary kernel too
    d, meta, parts, scales, (rp, re, rv) = _a2c_case(name)
    bf16 = d['logit'].dtype == BF16
    M = rp.size
    record = ops.ppo_hint(torch.device(DEV, torch.cuda.current_device()), 'a2c')  # the record the calls read
    saved = record.clone()
    worst = 0.0
    WORST.clear()
    try:
        ones = np.ones(M)
        r32, r64 = _a2c_refs(parts, A2C_RECORD, ones)
        for dd in (r32, r64):
            dd.pop('grad_logit'), dd.pop('grad_value')
        worst = compare_regimes(name + ' nograd', _a2c_run(d, A2C_RECORD, ones, bf16, None, grad=False)[0], r32, r64,
                                meta, scales)
        for mix in A2C_MIXES:
            keep_logit = _bits(mix[0], A2C_RECORD[0]) and _bits(mix[2], A2C_RECORD[2])
            keep_value = keep_logit and _bits(mix[1], A2C_RECORD[1])
            for path, poison, twice in (('poisoned', True, False), ('', False, False), ('twice', False, True)):
                mult = 2.0 if twice else 1.0
                div = row_divisor((abs(mix[0]) * rp + abs(mix[2]) * re) * mult / M)
                r32, r64 = _a2c_refs(parts, mix, div, mult)
                record.copy_(torch.tensor(list(A2C_RECORD) + [0.0]))
                got, gx, gv = _a2c_run(d, mix, div, bf16, r64['grad_logit'] * div[:, None], poison, twice)
                if poison and keep_logit:  # the backward returned without touching d logit: the forward's buffer
                    assert bool((gx == POISON).all()), (name, mix)
                    for dd in (got, r32, r64):
                        dd.pop('grad_logit')
                if poison and keep_value:
                    assert bool((gv == POISON).all()), (name, mix)
                    for dd in (got, r32, r64):
                        dd.pop('grad_value')
                elif poison:
                    assert not bool((gv == POISON).any()), (name, mix, 'd value not rewritten')
                worst = max(worst, compare_regimes('%s mix %s %s' % (name, mix, path), got, r32, r64, meta, scales))
    finally:
        record.copy_(saved)
    print('[fp64] %s worst %.2f  per regime %s' % (name, worst, _per_regime()))


# ----------------------------------------------------------------------------------------------------------------
# rows whose ratio overflows fp32 (not fp64): the non-finite pattern of the fp32 yardstick
# ----------------------------------------------------------------------------------------------------------------
def gen_overflow(seed, B, S, V, dtype, kind):
    """half the rows with lp_new - lp_old in (95, 110): exp overflows fp32 (> 88.7) but not fp64; the rest plain"""
    d, meta = gen_lm(seed, kind, B, S, V, dtype, 'frac', names=('plain', ))
    g = torch.Generator().manual_seed(seed + 2)
    rows = B * S
    ov = torch.rand(rows, generator=g) < 0.5
    old = d['logit_old'].float().reshape(rows, V)
    a = d['action'].reshape(-1)
    drop = 100.0 + 15.0 * torch.rand(rows, generator=g)
    old[torch.arange(rows)[ov], a[ov]] = old[ov].max(1).values - drop[ov]
    d['logit_old'] = old.to(dtype).reshape(B, S, V)
    return d, ov.numpy()


def _overflow_case(seed, dtype, kind):
    """gen_overflow on (4, 9, 1027) with overflow rows under a zero, a positive and a negative advantage (ratio * adv is
    then NaN, +inf and -inf): GRPO's sequence 0 has adv = 0, and PPO's first three rows get adv 0, 1, -1"""
    d, ov = gen_overflow(seed, 4, 9, 1027, dtype, kind)
    if kind == 'grpo':
        assert float(d['adv'][0]) == 0.0 and ov[:9].any() and (ov[9:] & (np.repeat(d['adv'].numpy(), 9)[9:] > 0)).any()
        assert (ov & (np.repeat(d['adv'].numpy(), 9) < 0)).any()
    else:
        d['adv'].view(-1)[:3] = torch.tensor([0.0, 1.0, -1.0])
        assert ov[:3].all(), 'reseed: the first three rows must overflow'
    return d, ov


OVERFLOW_CASES = {'grpo_f32': ('grpo', F32), 'grpo_bf16': ('grpo', BF16), 'ppo_f32': ('ppo_kl', F32),
                  'ppo_bf16': ('ppo_kl', BF16)}
OVERFLOW_SEEDS = {'grpo_f32': 9994, 'grpo_bf16': 9995, 'ppo_f32': 10024, 'ppo_bf16': 10065}  # each draws all three


def _overflow_refs(kind, d, dt):
    if kind == 'grpo':
        r = go.run64(d, dtype=dt)
        B, S, V = d['logit_new'].shape
        grad = torch.stack([go.grad_rows64(d['logit_new'][b], d['action'][b], r['dlp'][b], dt) for b in range(B)])
        return OrderedDict([('out_loss', r['loss']), ('out_approx_kl', r['approx_kl']),
                            ('grad_logit_new', _np(grad.reshape(B * S, V)))])
    r = po.run64(d, dual_clip=2.0, kl_type='k3', entropy_bonus=True, mix=PPO_MIX, dtype=dt)
    return OrderedDict([('out_policy', r['policy']), ('out_approx_kl', r['approx_kl']),
                        ('grad_logit_new', _np(r['grad'].reshape(-1, r['grad'].shape[-1])))])


@pytest.mark.gpu
@pytest.mark.parametrize('name', list(OVERFLOW_CASES))
def test_overflow_rows_match_the_fp32_pattern(name):
    kind, dtype = OVERFLOW_CASES[name]
    d, ov = _overflow_case(OVERFLOW_SEEDS[name], dtype, kind)
    d = _to(d, DEV)
    r32 = _overflow_refs(kind, d, torch.float32)
    ones = np.ones(ov.size)
    if kind == 'grpo':
        got = _gr_run(kind, d, ones, False, None, True)
        got = OrderedDict((k, got[k]) for k in r32)
    else:
        got = _ppo_run(d, dict(dual_clip=2.0, kl_type='k3', entropy_bonus=True), PPO_MIX, ones, False, None)
        got = OrderedDict((k, got[k]) for k in r32)
    gr = np.asarray(got['grad_logit_new']).reshape(ov.size, -1)
    assert not np.isfinite(np.asarray(r32['grad_logit_new']).reshape(ov.size, -1)[ov]).all()
    # the gradient's pattern of finite entries (where an overflowed row meets its one-hot entry the reference adds inf and
    # -inf to NaN, the kernel's c * (1 - p) is inf: both non-finite); the scalars' NaN and inf patterns exactly
    for k in r32:
        a, b = np.asarray(got[k], np.float64), np.asarray(r32[k], np.float64)
        assert np.array_equal(np.isfinite(a), np.isfinite(b)), (name, k, 'non-finite pattern')
        if not k.startswith('grad_'):
            assert np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(np.isposinf(a), np.isposinf(b)), \
                (name, k, 'NaN / inf pattern')
    assert np.isfinite(gr[~ov]).all()


# ----------------------------------------------------------------------------------------------------------------
# CPU: the regimes are what they claim, the rule is per regime, the fp32 restatement is the reference's arithmetic
# ----------------------------------------------------------------------------------------------------------------
def test_regime_checks_are_real():
    for V, dtype, rows in ((56333, F32, 133), (112648, BF16, 67), (112647, BF16, 67), (1027, F32, 529)):
        new, old, ref, action, meta = gen_rows(9001, rows, V, dtype)
        reg, names = meta['regime'], meta['names']
        frac = {nm: float(np.mean(reg == i)) for i, nm in enumerate(names)}
        assert min(frac.values()) >= 0.08, frac
        r = torch.arange(rows)

        def sel(nm):
            return torch.from_numpy(reg == names.index(nm))

        on = sel('onpolicy')
        assert torch.equal(new[on].view(torch.int16 if dtype == BF16 else torch.int32),
                           old[on].view(torch.int16 if dtype == BF16 else torch.int32))
        taken = new[r, action]
        assert torch.isfinite(taken[sel('masked')]).all() and torch.isfinite(old[r, action]).all()
        m = sel('masked')
        assert (~torch.isfinite(new[m]) | (new[m] <= -9000)).any(1).all()
        only = torch.from_numpy(meta['only'])
        assert only.any() and (torch.isfinite(new[only]).sum(1) == 1).all()
        lp = torch.from_numpy(_lp64(new, action))
        pk = sel('peaked')
        assert ((lp[pk] > -1e-8) | (lp[pk] < -20)).all()
        take = torch.from_numpy(meta['peaked_take'])
        assert (lp[take] > -1e-8).all() and (lp[pk & ~take] < -20).all()
        fl = sel('flat')
        assert torch.allclose(lp[fl], torch.full((int(fl.sum()), ), -math.log(V), dtype=torch.float64), rtol=0,
                              atol=1e-12)
        far = sel('far')
        ratio = torch.exp(lp - torch.from_numpy(_lp64(old, action)))
        assert ((ratio[far] > 1.2) | (ratio[far] < 0.8)).double().mean() >= 0.8
        assert (lp - torch.from_numpy(_lp64(old, action))).abs().max() <= 60
        kf = sel('kl_far')
        up = torch.from_numpy(_lp64(ref, action))[kf] - lp[kf]
        assert up.median() >= 15 and up.max() >= 19
        # placements: head / tail / cache edge / uncached by the row's own alignment
        h, tail0, cend = row_layout(rows, V, meta['esize'])
        pl, a = meta['place'], action
        for c, test in (('head', a < h), ('tail', a >= tail0), ('zero', a == 0), ('last', a == V - 1),
                        ('uncached', (a >= cend) & (a < tail0)), ('cache_edge', (a - cend).abs() <= 1)):
            m = torch.from_numpy(pl == PLACES.index(c))
            avail = {'head': (h > 0).any(), 'tail': (tail0 < V).any(), 'uncached': (cend < tail0).any(),
                     'cache_edge': (cend < tail0).any()}.get(c, True)
            assert m.any() == bool(avail), c
            assert test[m].all(), c
        mh = torch.from_numpy(meta['mplace'] == 2) & ~sel('peaked') & ~sel('flat') & ~sel('masked') & ~sel('kl_far')
        assert mh.any() == bool((h > 0).any()) and (new[mh].float().argmax(1) < h[mh]).all()
        mt = torch.from_numpy(meta['mplace'] == 3) & ~sel('peaked') & ~sel('flat') & ~sel('masked') & ~sel('kl_far')
        assert mt.any() == bool((tail0 < V).any()) and (new[mt].float().argmax(1) >= tail0[mt]).all()
    # the overflow regime overflows fp32 and not fp64
    d, ov = gen_overflow(9990, 4, 9, 1027, F32, 'grpo')
    a = d['action'].reshape(-1)
    d32 = go.logp64(d['logit_new'].reshape(36, -1), a, F32) - go.logp64(d['logit_old'].reshape(36, -1), a, F32)
    d64 = _lp64(d['logit_new'], d['action']) - _lp64(d['logit_old'], d['action'])
    assert torch.isinf(torch.exp(d32[torch.from_numpy(ov)])).all()
    assert np.isfinite(np.exp(d64[ov])).all() and ov.any()
    # every overflow case has an overflowed row under adv = 0 (ratio * adv = NaN: the fp32 loss is NaN) and others
    for name, (kind, dtype) in OVERFLOW_CASES.items():
        d, ov = _overflow_case(OVERFLOW_SEEDS[name], dtype, kind)
        r32 = _overflow_refs(kind, d, torch.float32)
        assert math.isnan(r32['out_loss' if kind == 'grpo' else 'out_policy']), name


def test_the_rule_is_per_regime():
    """an error on one regime's rows that the whole-tensor scale absorbs is rejected by the per-regime check"""
    d, meta = gen_lm(9002, 'grpo', 4, 33, 300, F32, 'frac')
    B, S, V = d['logit_new'].shape
    r64 = go.run64(d)
    r32 = go.run64(d, dtype=torch.float32)
    lse64 = torch.logsumexp(d['logit_new'].double(), -1).reshape(-1).numpy()
    lse32 = torch.logsumexp(d['logit_new'], -1).reshape(-1).double().numpy()
    res64, res32 = OrderedDict(lse=lse64), OrderedDict(lse=lse32)
    compare_regimes('exact', OrderedDict(lse=lse64.copy()), res32, res64, meta)
    # the plain rows (lse ~ 8): move them by twice the bound of the whole tensor's largest lse (the x30 rows), far past
    # their own
    pk = meta['regime'] == meta['names'].index('plain')
    bad = lse64.copy()
    big = np.abs(lse64).max()
    assert big > 10 * np.abs(lse64[pk]).max()
    bad[pk] += 2 * EPS32 * big
    whole = max(float(np.abs(lse32 - lse64).max()), EPS32 * big)
    assert np.abs(bad - lse64).max() <= K * whole  # the whole-tensor rule would pass it
    with pytest.raises(AssertionError):
        compare_regimes('perturbed', OrderedDict(lse=bad), res32, res64, meta)
    # and a gradient row with a small coefficient, behind the large ones of the other rows
    grad64 = go.grad_rows64(d['logit_new'].reshape(-1, V), d['action'].reshape(-1), r64['dlp'].reshape(-1)).numpy()
    grad32 = go.grad_rows64(d['logit_new'].reshape(-1, V), d['action'].reshape(-1), r32['dlp'].reshape(-1),
                            torch.float32).double().numpy()
    div = row_divisor(r64['scale'].numpy())
    small = int(np.argmin(np.where(div > 0, div, np.inf)))
    badg = grad64.copy()
    badg[small] += 2 * EPS32 * np.abs(grad64).max()
    assert np.abs(badg - grad64).max() <= K * max(np.abs(grad32 - grad64).max(), EPS32 * np.abs(grad64).max())
    with pytest.raises(AssertionError):
        compare64('scaled row', OrderedDict(grad_x=badg / div[:, None]), OrderedDict(grad_x=grad32 / div[:, None]),
                  OrderedDict(grad_x=grad64 / div[:, None]))


def test_fp32_restatement_matches_the_reference():
    """the float32 restatements against the reference's own fp32 arithmetic on the same fp32 inputs"""
    from oracle import ref_lm, ref_loader
    if not ref_lm.available():
        pytest.skip('reference not importable here')
    with ref_lm.modules() as ref:
        for kind in ('grpo', 'rloo'):
            d, _ = gen_lm(9003, kind, 4, 9, 1027, F32, 'frac', K=2)
            x = d['logit_new'].clone().requires_grad_(True)
            if kind == 'grpo':
                loss, info = ref['grpo'].grpo_policy_error(ref['grpo'].grpo_policy_data(
                    x, d['logit_old'], d['logit_ref'], d['action'], d['adv'], d['weight']))
            else:
                loss, info = ref['rloo'].rloo_policy_error(ref['rloo'].rloo_policy_data(
                    x, d['logit_old'], d['action'], d['reward'], d['weight']))
            loss.backward()
            r32 = go.run64(d, dtype=torch.float32)
            r64 = go.run64(d)
            g32 = torch.stack([go.grad_rows64(d['logit_new'][b], d['action'][b], r32['dlp'][b], torch.float32)
                               for b in range(4)])
            g64 = torch.stack([go.grad_rows64(d['logit_new'][b], d['action'][b], r64['dlp'][b]) for b in range(4)])
            # the reference's own fp32 error is within the bound the restatement's sets: a fair yardstick
            for got, want, exact in ((r32['loss'], loss.item(), r64['loss']),
                                     (r32['approx_kl'], info.approx_kl, r64['approx_kl'])):
                assert _fair(want, got, exact, abs(exact)), (kind, got, want, exact)
            assert r32['clipfrac'] == info.clipfrac
            assert _fair(x.grad, g32, g64, float(g64.abs().max())), kind
    if not ref_loader.available():
        return
    from tests.golden.make_ppo_lm_golden import reference_call
    d, _ = gen_lm(9004, 'ppo_kl', 3, 7, 1027, F32, 'mask')
    pol, e, kl, akl, cf, grad = reference_call(ref_loader.load(), d, 2.0, 'k3', True)
    r32 = po.run64(d, dual_clip=2.0, kl_type='k3', entropy_bonus=True, dtype=torch.float32)
    r64 = po.run64(d, dual_clip=2.0, kl_type='k3', entropy_bonus=True)
    for k, v in (('policy', pol), ('entropy', e), ('kl', kl), ('approx_kl', akl)):
        assert _fair(v, r32[k], r64[k], abs(r64[k])), (k, r32[k], v, r64[k])
    assert r32['clipfrac'] == cf
    assert _fair(grad, r32['grad'], r64['grad'], float(r64['grad'].abs().max()))


def _fair(ref, r32, r64, scale):
    """the reference's fp32 error against fp64 within K times the restatement's (or 2^-24 * scale)"""
    e_ref, e32 = (float((torch.as_tensor(v).double() - torch.as_tensor(r64).double()).abs().max()) for v in (ref, r32))
    return e_ref <= K * max(e32, EPS32 * scale)
