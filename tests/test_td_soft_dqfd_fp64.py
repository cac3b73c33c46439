"""The DQfD, R2D3-sequence, Munchausen-DQN, soft Q-learning and discrete-SAC kernels against a float64 reference, at every
hand-off of the TD row plan they share with q-n-step (csrc/td.cu ``launch_td_rows``).

Kernels: ``dqfd_fwd_kernel`` / ``dqfd_bwd_kernel`` (dqfd_nstep_td_error, _with_rescale and R2D3's sequence form with its
priority) and ``soft_td_fwd_kernel`` modes 0 / 1 / 2 (m_q_1step_td_error, q_nstep_sql_td_error, q_v_1step_td_error) with
``qntd_bwd_kernel`` behind them.  Their loss sums run in the CTA (up to 1024 rows), through the one-round-trip
``grid_sum_fx`` (1025 - 65408 rows) or the ticketed ``grid_sum`` (more rows, or any sequence priority): the row counts
below sit on both sides of every one of those hand-offs (and of 256 / 512 threads), and of the 4-wide margin unroll and
the n-step tail loop past 8 rewards.

Each row is drawn from one of several regimes in equal shares: live / terminal / fractional / non-binary ``done`` (and,
drawn on its own, ``done_one_step``), zero weights, rows exactly on the criterion's edge, exact margin ties (dyadic q with
q_j + margin == q_a, and two j tied), the Munchausen clamp at exactly +-1 (tau = +-1/256 on a 0.25 grid), top-1 == top-2,
near-deterministic next policies, infinite soft values, and rows whose 128-row tile sums exceed 2^36.

Reference: ``tests/dqfd_oracle.py`` and ``tests/soft_td_oracle.py`` (bit-exact restatements of the reference in fp32) on
float64 copies of the inputs, with float64 as torch's default dtype.  The fp32 oracle on the fp32 inputs is the yardstick
(``test_offpolicy_fp64.compare64``):  max|X_gpu - X_64| <= K * max(max|X_32 - X_64|, 2^-24 * scale_X)  for every output and
the gradient of q, over the whole tensor and again over the rows of each regime, for a unit upstream gradient (the
gradient the forward launch wrote) and for an upstream mix through the backward launch; each GPU run happens twice.
Rows on a discontinuity that fp32 rounding may cross (a near-tie of the margin max that is not exact, an L1 row with
0 < |d| < 1e-5, a Munchausen log-policy within rounding of +-1) are left out of the elementwise gradient check and the
clip flags, but must be finite.
"""
import functools
from collections import OrderedDict

import numpy as np
import pytest
import torch
import torch.nn as nn

from oracle import rl_oracle
from tests import cases
from tests import dqfd_oracle as dqo
from tests import soft_td_oracle as sto
from tests.test_offpolicy_fp64 import EPS32, K, compare64
from tests.test_value_td_fp64 import (CRITERIA, SANE, _dyadic, _per_upstream, _regimes, _value_gamma, _zeros_at,
                                      float64_default, gen_qn, gen_qt, to64)

assert K == 8.0  # the bound of the PPO-family fp64 suite, shared, not loosened here
DEV = 'cuda'
REGIME_MIN = 0.02
MIX = dict(loss=0.7, s_n=0.7, s_1=-0.4, s_je=1.9)  # upstream gradients of the backward-launch run
DONE_KINDS = ('live', 'terminal', 'fractional', 'nonbinary')
HUGE = (5.5, 6.5)  # log10 |q_sa - target| of the large-magnitude rows: 16 of them put a 128-row tile above 2^36


# ----------------------------------------------------------------------------------------------------------------
# row regimes
# ----------------------------------------------------------------------------------------------------------------
def _done_of(g, kind):
    """done per row from its kind (index into DONE_KINDS)"""
    n = kind.shape[0]
    d = torch.zeros(n)
    d[kind == 1] = 1.0
    d[kind == 2] = torch.rand(n, generator=g)[kind == 2]
    d[kind == 3] = (3.0 * torch.randn(n, generator=g))[kind == 3]
    return d


def _row_done(g, reg, names):
    """done from the row's regime where it is a done regime, a random kind elsewhere"""
    kind = torch.randint(0, 4, reg.shape, generator=g)
    for i, nm in enumerate(names):
        if nm in DONE_KINDS:
            kind[reg == i] = DONE_KINDS.index(nm)
    return _done_of(g, kind)


def _huge(g, n, rng=HUGE):
    mag = 10.0 ** (torch.rand(n, generator=g) * (rng[1] - rng[0]) + rng[0])
    return torch.where(torch.rand(n, generator=g) < 0.5, -mag, mag)


# ----------------------------------------------------------------------------------------------------------------
# DQfD (dqfd_fwd_kernel / dqfd_bwd_kernel)
# ----------------------------------------------------------------------------------------------------------------
def gen_dqfd(seed, S, N, nstep, crit='mse', vg=None, expert='float', cum=False, rescale=False, lam=(1.0, 1.0, 1.0),
             margin=0.5, huge=False, T=None, mix=0.9):
    """``S`` rows (``T`` * B in the sequence form).  edge: done = done_one_step = 1, one dyadic reward, q_sa on the
    criterion's edge from it; tie: q on a 0.25 grid (q_j + margin ties q_a, or another j); huge: |q_sa - target| ~ 1e6."""
    g = cases._g(seed)
    names = DONE_KINDS + ('zero_w', 'tie') + (() if rescale else ('edge', )) + (('huge', ) if huge else ())
    reg = _regimes(g, S, names)
    pick = {nm: reg == i for i, nm in enumerate(names)}
    done = _row_done(g, reg, names)
    done1 = _done_of(g, torch.randint(0, 4, (S, ), generator=g))
    q = torch.randn(S, N, generator=g)
    act = torch.randint(0, N, (S, ), generator=g)
    tie = pick['tie']
    q[tie] = torch.randint(0, 4, (int(tie.sum()), N), generator=g).float() * 0.25
    if N > 1:  # every other tie row: q_a == max_{j != a} q_j + margin, the action tied with the margin maximum
        ta = torch.nonzero(tie).reshape(-1)[::2]
        other = q[ta].clone()
        other[torch.arange(ta.numel()), act[ta]] = -1e9
        q[ta, act[ta]] = other.max(1)[0] + margin
    if rescale:  # h^-1 of next values from 1e-3 to ~1e5
        mags = [10.0 ** (torch.rand(S, N, generator=g) * 8.0 - 3.0) for _ in range(2)]
        nq, nq1 = (torch.where(torch.rand(S, N, generator=g) < 0.5, -m, m) for m in mags)
    else:
        nq, nq1 = torch.randn(S, N, generator=g), torch.randn(S, N, generator=g)
    reward = torch.rand(nstep, S, generator=g) * 2.0 - 1.0
    if 'edge' in pick:
        e = pick['edge']
        r0 = _dyadic(g, S)
        done[e] = 1.0
        done1[e] = 1.0
        reward[:, e] = 0.0
        reward[0, e] = r0[e]
        sign = torch.where(torch.rand(S, generator=g) < 0.5, -1.0, 1.0)
        q[e, act[e]] = (r0 + sign * CRITERIA[crit][1])[e]
    if huge:  # True, or the log10 range of |q_sa - target|
        h = pick['huge']
        q[h, act[h]] += _huge(g, S, HUGE if huge is True else huge)[h]
    weight = _zeros_at(g, torch.rand(S, generator=g) + 0.25, 0.02)
    weight[pick['zero_w']] = 0.0
    ie = torch.randint(0, 2, (S, ), generator=g)
    ie = {'float': ie.float(), 'int': ie, 'bool': ie.bool()}[expert]
    t = OrderedDict()
    p = dict(gamma=0.97, nstep=nstep, lam=tuple(lam), margin=margin, rescale=rescale, crit=crit)
    if T is None:
        t['q'], t['next_n_q'], t['action'] = q, nq, act
        t['next_n_action'] = torch.randint(0, N, (S, ), generator=g)
        t['reward'] = reward[0] if cum else reward
        t['done'], t['done_one_step'], t['weight'] = done, done1, weight
        t['new_n_q_one_step'] = nq1
        t['next_n_action_one_step'] = torch.randint(0, N, (S, ), generator=g)
        t['is_expert'] = ie
        p['cum'] = cum
        _value_gamma(g, vg, S, t, p)
        op = 'dqfd'
    else:
        B = S // T
        lead = (T, B)
        t['q'], t['next_n_q'], t['action'] = q.reshape(T, B, N), nq.reshape(T, B, N), act.reshape(lead)
        t['next_n_action'] = torch.randint(0, N, lead, generator=g)
        t['reward'] = reward.reshape(nstep, T, B).permute(1, 0, 2).contiguous()
        t['done'], t['done_one_step'], t['weight'] = done.reshape(lead), done1.reshape(lead), weight.reshape(lead)
        t['new_n_q_one_step'] = nq1.reshape(T, B, N)
        t['next_n_action_one_step'] = torch.randint(0, N, lead, generator=g)
        t['is_expert'] = ie.reshape(lead)
        if vg == 'tensor':
            t['value_gamma'] = (torch.rand(S, generator=g) * 0.2 + 0.8).reshape(lead)
        p['priority_mix'] = mix
        op = 'dqfd_seq'
    return op, t, p, dict(regime=reg.numpy(), names=names, R=S)


# ----------------------------------------------------------------------------------------------------------------
# Munchausen DQN (soft_td_fwd_kernel mode 0)
# ----------------------------------------------------------------------------------------------------------------
GRID_OFF = torch.tensor([0.0, -0.5, -1.0, -1.25, -1.75, -2.25, -2.75, -3.25])


def gen_mdqn(seed, S, N, tau, crit='mse', alpha=0.5, huge=False):
    """grid: target_q distinct on a 0.25 grid, >= 0.5 from the row's max (tau > 0) or min (tau < 0): with |tau| = 1/256
    log pi(a) is exactly x_a - x_max (or - x_min), and +-1 is hit; edge: a grid row with done 1, a dyadic reward, and q_sa
    on the criterion's edge from the (exact) target; tie: top-1 == top-2; peaked: next_q x 60, so that the next policy's
    exp underflows for every action but one."""
    g = cases._g(seed)
    exact = abs(tau) == 1 / 256
    names = DONE_KINDS + ('zero_w', 'tie', 'peaked') + (('grid', 'edge') if exact and N <= 8 else ()) + \
        (('huge', ) if huge else ())
    reg = _regimes(g, S, names)
    pick = {nm: reg == i for i, nm in enumerate(names)}
    done = _row_done(g, reg, names)
    q = torch.randn(S, N, generator=g)
    tq = torch.randn(S, N, generator=g)
    nq = torch.randn(S, N, generator=g)
    act = torch.randint(0, N, (S, ), generator=g)
    reward = torch.randn(S, generator=g)
    sgn = 1.0 if tau > 0 else -1.0
    for nm in ('grid', 'edge'):
        if nm in pick:
            m = pick[nm]
            n = int(m.sum())
            rows = torch.stack([GRID_OFF[:N][torch.randperm(N, generator=g)] for _ in range(n)]) * sgn
            tq[m] = rows + torch.randint(-3, 4, (n, 1), generator=g).float()
    if 'edge' in pick:
        e = pick['edge']
        r0 = _dyadic(g, S)
        done[e] = 1.0
        reward[e] = r0[e]
        lp = tq - (tq.max(1, keepdim=True)[0] if tau > 0 else tq.min(1, keepdim=True)[0])
        target = r0 + alpha * lp.gather(1, act.reshape(S, 1)).reshape(S).clamp(-1, 1)
        sign = torch.where(torch.rand(S, generator=g) < 0.5, -1.0, 1.0)
        q[e, act[e]] = (target + sign * CRITERIA[crit][1])[e]
    m = pick['tie']
    top = tq.argsort(1, descending=True)
    tq[m, top[m, 1]] = tq[m, top[m, 0]]
    nq[pick['peaked']] *= 60.0
    if huge:
        h = pick['huge']
        q[h, act[h]] += _huge(g, S)[h]
    weight = _zeros_at(g, torch.rand(S, generator=g) + 0.25, 0.02)
    weight[pick['zero_w']] = 0.0
    t = OrderedDict(q=q, target_q=tq, next_q=nq, act=act, reward=reward, done=done, weight=weight)
    return 'mdqn', t, dict(gamma=0.97, tau=tau, alpha=alpha, crit=crit), dict(regime=reg.numpy(), names=names, R=S)


# ----------------------------------------------------------------------------------------------------------------
# soft Q-learning (mode 1)
# ----------------------------------------------------------------------------------------------------------------
def gen_sql(seed, S, N, nstep, alpha, crit='mse', vg=None, cum=0, huge=False, nan=False):
    """inf: next_n_q rows holding +inf, -inf, both (V' = +-20), and with ``nan`` also a NaN (V' NaN); edge: done 1, one dyadic reward, q_sa on the edge;
    cum: 0 off, 1 a (S,) reward, K > 1 a (K, S) reward (the error broadcasts to (K, S))"""
    g = cases._g(seed)
    names = DONE_KINDS + ('zero_w', 'inf') + (('edge', ) if not cum else ()) + (('huge', ) if huge else ())
    reg = _regimes(g, S, names)
    pick = {nm: reg == i for i, nm in enumerate(names)}
    done = _row_done(g, reg, names)
    q = torch.randn(S, N, generator=g)
    nq = torch.randn(S, N, generator=g) * 3.0
    act = torch.randint(0, N, (S, ), generator=g)
    m = torch.nonzero(pick['inf']).reshape(-1)
    kind = torch.randint(0, 4 if nan else 3, (m.numel(), ), generator=g)
    col = torch.randint(0, N, (m.numel(), ), generator=g)
    for r, k, c in zip(m.tolist(), kind.tolist(), col.tolist()):
        if k == 0:
            nq[r, c] = float('inf')
        elif k == 1:
            nq[r, :] = float('-inf')
        elif k == 3:
            nq[r, c] = float('nan')
        else:
            nq[r, c] = float('inf')
            nq[r, (c + 1) % N] = float('-inf')
    reward = torch.rand(cum if cum > 1 else (1 if cum else nstep), S, generator=g)
    if 'edge' in pick:
        e = pick['edge']
        r0 = _dyadic(g, S)
        done[e] = 1.0
        reward[:, e] = 0.0
        reward[0, e] = r0[e]
        sign = torch.where(torch.rand(S, generator=g) < 0.5, -1.0, 1.0)
        q[e, act[e]] = (r0 + sign * CRITERIA[crit][1])[e]
    if huge:
        h = pick['huge']
        q[h, act[h]] += _huge(g, S)[h]
    wshape = (cum, S) if cum > 1 else (S, )
    weight = _zeros_at(g, torch.rand(wshape, generator=g) + 0.25, 0.02)
    weight[..., pick['zero_w']] = 0.0
    t = OrderedDict(q=q, next_n_q=nq, action=act, next_n_action=torch.randint(0, N, (S, ), generator=g),
                    reward=reward[0] if cum == 1 else reward, done=done, weight=weight)
    p = dict(gamma=0.97, alpha=alpha, nstep=nstep, cum=bool(cum), crit=crit)
    _value_gamma(g, vg, S, t, p)
    return 'sql', t, p, dict(regime=reg.numpy(), names=names, R=S)


# ----------------------------------------------------------------------------------------------------------------
# discrete SAC critic (mode 2)
# ----------------------------------------------------------------------------------------------------------------
def gen_qv(seed, B, N, A=None, wshape='full', crit='mse', huge=False):
    """A: None for q (B, N), else q (B, A, N) (reward and done broadcast over the agents); wshape 'full' or 'col' ((B, 1))"""
    g = cases._g(seed)
    names = DONE_KINDS + ('zero_w', 'edge') + (('huge', ) if huge else ())
    reg = _regimes(g, B, names)
    pick = {nm: reg == i for i, nm in enumerate(names)}
    done = _row_done(g, reg, names)
    lead = (B, ) if A is None else (B, A)
    q = torch.randn(*lead, N, generator=g)
    v = torch.randn(*lead, generator=g)
    act = torch.randint(0, N, lead, generator=g)
    reward = torch.randn(B, generator=g)
    qv, av = q.reshape(B, -1, N), act.reshape(B, -1)
    e = pick['edge']
    r0 = _dyadic(g, B)
    done[e] = 1.0
    reward[e] = r0[e]
    sign = torch.where(torch.rand(B, generator=g) < 0.5, -1.0, 1.0)
    for j in range(qv.shape[1]):
        qv[e, j, av[e, j]] = (r0 + sign * CRITERIA[crit][1])[e]
        if huge:
            h = pick['huge']
            qv[h, j, av[h, j]] += _huge(g, B)[h]
    weight = _zeros_at(g, torch.rand(*(lead if wshape == 'full' else (B, 1)), generator=g) + 0.25, 0.02)
    weight[pick['zero_w']] = 0.0
    t = OrderedDict(q=q, v=v, act=act, reward=reward, done=done, weight=weight)
    return 'qv', t, dict(gamma=0.97, crit=crit), dict(regime=reg.numpy(), names=names, R=B)


# ----------------------------------------------------------------------------------------------------------------
# one call of a loss: the package on the GPU ('gpu') or the restated reference ('ref', in the inputs' dtype)
# ----------------------------------------------------------------------------------------------------------------
def _crit(name, record=None):
    c = CRITERIA[name][0]()
    if record is None:
        return c

    class Recording(nn.Module):
        reduction = 'none'

        def forward(self, x, y):
            record.append((x - y).detach().reshape(-1).double().numpy())
            return c(x, y)

    return Recording()


def call(op, impl, t, p, path, record=None, dtypes=None):
    """-> OrderedDict of float64 numpy results: out_* outputs and grad_q; ``dtypes`` (a dict) receives the torch dtype of
    each before the conversion"""
    import di_engine_b200 as b2
    dev = DEV if impl == 'gpu' else 'cpu'
    d = OrderedDict((k, v.to(dev) if isinstance(v, torch.Tensor) else v) for k, v in t.items())
    q = d['q'].clone().requires_grad_(True)
    vg = d.get('value_gamma', p.get('value_gamma'))
    crit = _crit(p.get('crit', 'mse'), record)
    out = OrderedDict()
    if op in ('dqfd', 'dqfd_seq'):
        ln, ls, l1 = p['lam']
        ops_ = [q] + [d[k] for k in ('next_n_q', 'action', 'next_n_action', 'reward', 'done', 'done_one_step', 'weight',
                                     'new_n_q_one_step', 'next_n_action_one_step', 'is_expert')]
        if op == 'dqfd_seq':
            if impl == 'gpu':
                res = b2.dqfd_nstep_td_error_sequence(b2.dqfd_nstep_td_seq_data(*ops_), p['gamma'], ln, ls, p['margin'], l1,
                                                      p['nstep'], value_gamma=vg, rescale=p['rescale'],
                                                      priority_mix=p['priority_mix'])
            else:
                res = dqo.dqfd_nstep_td_error_sequence(*ops_, p['gamma'], ln, ls, p['margin'], l1, p['nstep'], vg,
                                                       rescale=p['rescale'], priority_mix=p['priority_mix'])
            loss, prio, per, st = res
            out['out_priority'] = prio
        elif impl == 'gpu':
            data = b2.dqfd_nstep_td_data(*ops_)
            kw = dict(nstep=p['nstep'], cum_reward=p['cum'], value_gamma=vg, criterion=crit)
            if p['rescale']:
                loss, per, st = b2.dqfd_nstep_td_error_with_rescale(data, p['gamma'], ln, ls, l1, p['margin'], **kw)
            else:
                loss, per, st = b2.dqfd_nstep_td_error(data, p['gamma'], ln, ls, p['margin'], l1, **kw)
        else:
            loss, per, st = dqo.dqfd_nstep_td_error(*ops_, p['gamma'], ln, ls, p['margin'], l1, p['nstep'], p['cum'], vg,
                                                    crit, p['rescale'])
        out['out_loss'], out['out_per'] = loss, per
        out['out_s_n'], out['out_s_1'], out['out_s_je'] = st
        extra = MIX['s_n'] * st[0] + MIX['s_1'] * st[1] + MIX['s_je'] * st[2]
    else:
        api = b2.rl_utils if impl == 'gpu' else sto
        if op == 'mdqn':
            data = api.m_q_1step_td_data(q, *[d[k] for k in ('target_q', 'next_q', 'act', 'reward', 'done', 'weight')])
            loss, per, gap, clip = api.m_q_1step_td_error(data, p['gamma'], p['tau'], p['alpha'], crit)
            out['out_gap'], out['out_clip'] = gap, clip
        elif op == 'sql':
            data = api.q_nstep_td_data(q, *[d[k] for k in ('next_n_q', 'action', 'next_n_action', 'reward', 'done',
                                                           'weight')])
            loss, per, rec = api.q_nstep_sql_td_error(data, p['gamma'], p['alpha'], nstep=p['nstep'], cum_reward=p['cum'],
                                                      value_gamma=vg, criterion=crit)
            out['out_rec'] = rec
        else:
            data = api.q_v_1step_td_data(q, *[d[k] for k in ('v', 'act', 'reward', 'done', 'weight')])
            loss, per = api.q_v_1step_td_error(data, p['gamma'], crit)
        out['out_loss'], out['out_per'] = loss, per
        extra = 0.0
    if path == 'unit':
        loss.backward()
    else:
        up = _per_upstream(tuple(per.shape)).to(dtype=per.dtype, device=per.device)
        (MIX['loss'] * loss + (per * up).sum() + extra).backward()
    out['grad_q'] = q.grad
    if dtypes is not None:
        dtypes.update((k, v.dtype) for k, v in out.items())
    return OrderedDict((k, v.detach().cpu().numpy().astype(np.float64)) for k, v in out.items())


def run_ref(op, t, p, path):
    """(fp32 oracle, fp64 oracle, fp64 criterion differences, torch dtypes of the fp64 oracle's results)"""
    r32 = call(op, 'ref', t, p, path)
    rec, dtypes = [], {}
    with float64_default():
        r64 = call(op, 'ref', to64(t), p, path, record=rec, dtypes=dtypes)
    return r32, r64, rec, dtypes


# ----------------------------------------------------------------------------------------------------------------
# the cases
# ----------------------------------------------------------------------------------------------------------------
CASES = OrderedDict([
    # DQfD: one CTA of 256 / 512 / 1024 threads, grid_sum_fx from 1025 to 65408 rows, the ticketed sum above; N covers
    # the remainders of the 4-wide margin unroll; nstep 1 / 8 / 9 / 12
    ('dqfd_mse_n1_S1_N2', lambda: gen_dqfd(9001, 1, 2, 1)),
    ('dqfd_l1_n8_S256_N5_vgT', lambda: gen_dqfd(9002, 256, 5, 8, crit='l1', vg='tensor', expert='int')),
    ('dqfd_smoothl1_n9_S257_N1000_vg0', lambda: gen_dqfd(9003, 257, 1000, 9, crit='smoothl1', vg='0dim')),
    ('dqfd_huber_n12_S512_N18_vgF', lambda: gen_dqfd(9004, 512, 18, 12, crit='huber', vg='float', expert='bool')),
    ('dqfd_mse_n9_S513_N3_cum', lambda: gen_dqfd(9005, 513, 3, 9, cum=True, vg='tensor')),
    ('dqfd_l1_n1_S1024_N2_lamneg', lambda: gen_dqfd(9006, 1024, 2, 1, crit='l1', lam=(1.0, 0.8, -0.5))),
    ('dqfd_mse_n12_S1025_N5_vgT', lambda: gen_dqfd(9007, 1025, 5, 12, vg='tensor', lam=(0.9, -0.6, 1.1), margin=0.25)),
    ('dqfd_huber_n8_S65408_N3_cum', lambda: gen_dqfd(9008, 65408, 3, 8, crit='huber', cum=True, vg='float')),
    ('dqfd_smoothl1_n9_S65409_N1', lambda: gen_dqfd(9009, 65409, 1, 9, crit='smoothl1', expert='bool')),
    ('dqfd_mse_n12_S100003_N2_vgT', lambda: gen_dqfd(9010, 100003, 2, 12, vg='tensor', expert='int')),
    ('dqfdr_n9_S1025_N5_vgT', lambda: gen_dqfd(9011, 1025, 5, 9, rescale=True, vg='tensor')),
    ('dqfdr_huber_n1_S256_N18', lambda: gen_dqfd(9012, 256, 18, 1, rescale=True, crit='huber')),
    ('dqfdr_n12_S65409_N3_cum_lamneg', lambda: gen_dqfd(9013, 65409, 3, 12, rescale=True, cum=True, lam=(1.0, 1.0, -1.0))),
    # R2D3 sequence: one CTA (T*B <= 128), 129 rows, 511 / 512 CTAs, B > 128 columns per thread stride
    ('seq_T4_B32_mix0.9', lambda: gen_dqfd(9020, 128, 6, 5, T=4, vg='tensor', mix=0.9)),
    ('seq_T3_B43_mix0_rescale', lambda: gen_dqfd(9021, 129, 4, 9, T=3, rescale=True, vg='tensor', mix=0.0)),
    ('seq_T2_B32704_mix1', lambda: gen_dqfd(9022, 65408, 3, 8, T=2, mix=1.0, lam=(1.0, 1.0, -0.5))),
    ('seq_T3_B21803_mix0.9_rescale', lambda: gen_dqfd(9023, 65409, 2, 12, T=3, rescale=True, vg='tensor', mix=0.9)),
    # M-DQN
    ('mdqn_N2_S1', lambda: gen_mdqn(9030, 1, 2, 0.03)),
    ('mdqn_N6_S256_grid', lambda: gen_mdqn(9031, 256, 6, 1 / 256, crit='l1')),
    ('mdqn_N1000_S257', lambda: gen_mdqn(9032, 257, 1000, 0.03, crit='huber')),
    ('mdqn_N5_S512_gridneg', lambda: gen_mdqn(9033, 512, 5, -1 / 256, crit='smoothl1')),
    ('mdqn_N18_S513', lambda: gen_mdqn(9034, 513, 18, 0.03)),
    ('mdqn_N3_S1024_grid', lambda: gen_mdqn(9035, 1024, 3, 1 / 256, crit='huber')),
    ('mdqn_N6_S1025_gridneg', lambda: gen_mdqn(9036, 1025, 6, -1 / 256)),
    ('mdqn_N2_S65408', lambda: gen_mdqn(9037, 65408, 2, 0.03, crit='l1')),
    ('mdqn_N3_S65409_grid', lambda: gen_mdqn(9038, 65409, 3, 1 / 256, crit='smoothl1')),
    ('mdqn_N6_S100003', lambda: gen_mdqn(9039, 100003, 6, 0.03)),
    # soft Q-learning
    ('sql_a0.08_n1_S1', lambda: gen_sql(9040, 1, 4, 1, 0.08)),
    ('sql_a0.01_n8_S256_vgT', lambda: gen_sql(9041, 256, 6, 8, 0.01, crit='l1', vg='tensor')),
    ('sql_a1_n9_S257_N1000', lambda: gen_sql(9042, 257, 1000, 9, 1.0, crit='huber', vg='0dim')),
    ('sql_a5_n12_S512_vgF', lambda: gen_sql(9043, 512, 5, 12, 5.0, crit='smoothl1', vg='float')),
    ('sql_a0.08_S513_cum1', lambda: gen_sql(9044, 513, 4, 3, 0.08, cum=1, vg='tensor')),
    ('sql_a1_n9_S1024', lambda: gen_sql(9045, 1024, 3, 9, 1.0)),
    ('sql_a0.01_S1025_cumK3', lambda: gen_sql(9046, 1025, 4, 2, 0.01, cum=3, crit='huber')),
    ('sql_a5_n12_S65408_vgT', lambda: gen_sql(9047, 65408, 3, 12, 5.0, crit='l1', vg='tensor')),
    ('sql_a0.08_n8_S65409', lambda: gen_sql(9048, 65409, 2, 8, 0.08, vg='0dim')),
    ('sql_a1_n1_S100003_cumK2', lambda: gen_sql(9049, 100003 // 2, 2, 1, 1.0, cum=2)),
    ('sql_nan_a0.5_n3_S256', lambda: gen_sql(9062, 256, 4, 3, 0.5, nan=True)),
    ('sql_nan_a1_n9_S1025', lambda: gen_sql(9063, 1025, 3, 9, 1.0, nan=True, vg='tensor')),
    ('sql_nan_a0.08_n1_S100003', lambda: gen_sql(9064, 100003, 2, 1, 0.08, nan=True)),
    # discrete SAC: A = 1 at every row-count hand-off; A = 3 at B = 341 / 342 and 21802 / 21803
    ('qv_S1', lambda: gen_qv(9050, 1, 3)),
    ('qv_S256_l1', lambda: gen_qv(9051, 256, 6, crit='l1')),
    ('qv_S257_smoothl1', lambda: gen_qv(9052, 257, 6, crit='smoothl1')),
    ('qv_S512_huber', lambda: gen_qv(9053, 512, 4, crit='huber')),
    ('qv_S513', lambda: gen_qv(9054, 513, 4)),
    ('qv_A3_B341_wfull', lambda: gen_qv(9055, 341, 5, A=3)),
    ('qv_A3_B342_wcol_huber', lambda: gen_qv(9056, 342, 5, A=3, wshape='col', crit='huber')),
    ('qv_S1024_l1', lambda: gen_qv(9057, 1024, 2, crit='l1')),
    ('qv_S1025', lambda: gen_qv(9058, 1025, 2)),
    ('qv_A3_B21802_wcol', lambda: gen_qv(9059, 21802, 3, A=3, wshape='col')),
    ('qv_A3_B21803_wfull_l1', lambda: gen_qv(9060, 21803, 3, A=3, crit='l1')),
    ('qv_S100003_smoothl1', lambda: gen_qv(9061, 100003, 2, crit='smoothl1')),
    # rows whose 128-row tile sums exceed 2^36, at <= 1024 rows, on the one-round-trip sum and on the ticketed sum
    ('huge_dqfd_S1024', lambda: gen_dqfd(9070, 1024, 4, 3, huge=True)),
    ('huge_dqfd_S4099', lambda: gen_dqfd(9071, 4099, 4, 3, huge=True, lam=(1.0, 1.0, -0.5))),
    ('huge_dqfd_S65409', lambda: gen_dqfd(9072, 65409, 3, 9, huge=True)),
    ('huge_mdqn_S1024', lambda: gen_mdqn(9073, 1024, 4, 0.03, huge=True)),
    ('huge_mdqn_S4099', lambda: gen_mdqn(9074, 4099, 4, 0.03, huge=True)),
    ('huge_mdqn_S65409', lambda: gen_mdqn(9075, 65409, 3, 0.03, huge=True)),
    ('huge_sql_S1024', lambda: gen_sql(9076, 1024, 4, 3, 0.5, huge=True)),
    ('huge_sql_S4099', lambda: gen_sql(9077, 4099, 4, 9, 0.5, huge=True)),
    ('huge_sql_S65409', lambda: gen_sql(9078, 65409, 3, 3, 0.5, huge=True)),
    ('huge_qv_S1024', lambda: gen_qv(9079, 1024, 4, huge=True)),
    ('huge_qv_S4099', lambda: gen_qv(9080, 4099, 4, huge=True)),
    ('huge_qv_A3_S65409', lambda: gen_qv(9081, 21803, 3, A=3, huge=True)),
    # large NEGATIVE loss partials (lambda_1 < -lambda_n): CTA sums from about -2^36 to -2^43, where an inexact split of a
    # negative partial would lose bits that the fp32 oracle keeps
    ('huge_neg_dqfd_S1024', lambda: gen_dqfd(9082, 1024, 4, 3, huge=(4.8, 5.3), lam=(1.0, 0.5, -2.0))),
    ('huge_neg_dqfd_S4099', lambda: gen_dqfd(9083, 4099, 4, 3, huge=(4.8, 5.3), lam=(1.0, 0.5, -2.0))),
    ('huge_neg_dqfd_S65408', lambda: gen_dqfd(9084, 65408, 3, 9, huge=(4.8, 5.3), lam=(1.0, 0.5, -2.0), vg='tensor')),
    ('huge_neg_dqfd_S65409', lambda: gen_dqfd(9085, 65409, 3, 3, huge=(4.8, 5.3), lam=(1.0, 0.5, -2.0))),
])


# ----------------------------------------------------------------------------------------------------------------
# per-row views, boundary rows
# ----------------------------------------------------------------------------------------------------------------
def row_views(res, R):
    """every per-row output reshaped to (R, ...); the scalars and the priority (per batch column) as they are"""
    out = OrderedDict()
    for k, v in res.items():
        v = np.asarray(v)
        if k != 'out_priority' and v.ndim >= 1 and (v.shape[0] == R or (v.ndim >= 2 and v.shape[0] * v.shape[1] == R)):
            v = v.reshape((R, -1))
        out[k] = v
    return out


def _per_row_keys(views, R):
    return [k for k, v in views.items() if v.ndim == 2 and v.shape[0] == R and R > 1]


def boundary(op, t, p, meta, rec):
    """rows whose fp64 result sits on a discontinuity fp32 rounding may cross (see the module docstring)"""
    R = meta['R']
    bnd = np.zeros(R, bool)
    if p.get('crit') == 'l1':
        for d in rec:
            d = np.abs(d)
            near = (d > 0) & (d < 1e-5)
            bnd |= near.reshape(R, -1).any(1) if op == 'qv' else near.reshape(-1, R).any(0)
    if op in ('dqfd', 'dqfd_seq'):
        q = t['q'].double().reshape(R, -1).numpy()
        a = t['action'].reshape(R).numpy()
        x = q + p['margin']
        x[np.arange(R), a] = q[np.arange(R), a]
        if x.shape[1] > 1:
            top = -np.sort(-x, axis=1)[:, :2]
            gap = top[:, 0] - top[:, 1]
            bnd |= (gap > 0) & (gap <= 1e-5 * np.maximum(1.0, np.abs(top[:, 0])))
    return bnd


def clip_boundary(t, p):
    """M-DQN rows whose fp64 log pi(a) is within rounding of +-1 without being exactly +-1"""
    with float64_default():
        tq = t['target_q'].double()
        _, lp = sto._log_policy(tq, p['tau'])
        lp = lp.gather(1, t['act'].reshape(-1, 1)).reshape(-1).numpy()
    near = lambda e: (np.abs(lp - e) <= 1e-5) & (lp != e)  # noqa: E731
    return near(1.0) | near(-1.0)


def regime_fractions(meta):
    reg = meta['regime']
    return {nm: float(np.mean(reg == i)) for i, nm in enumerate(meta['names'])}


@functools.lru_cache(maxsize=2)
def _case(name):
    op, t, p, meta = CASES[name]()
    refs = {path: run_ref(op, t, p, path) for path in ('unit', 'mix')}
    return op, t, p, meta, refs


def compare_case(tag, op, t, p, meta, got, r32, r64, rec):
    R = meta['R']
    bnd = boundary(op, t, p, meta, rec)
    got, r32, r64 = (row_views(x, R) for x in (got, r32, r64))
    if 'out_clip' in r64:  # a per-row 0 / 1 flag: exact outside the rows on the clamp's edge
        cb = clip_boundary(t, p)
        x, b = got.pop('out_clip').reshape(-1), r64.pop('out_clip').reshape(-1)
        r32.pop('out_clip')
        assert np.array_equal(x[~cb], b[~cb]), (tag, 'clipfrac', int((x[~cb] != b[~cb]).sum()))
        assert cb.sum() <= 1e-3 * R + 1, (tag, 'clip boundary rows', int(cb.sum()))
    worst = compare64(tag, got, r32, r64, bnd=bnd if R > 1 else None, S=R)
    keys = _per_row_keys(r64, R)
    for i, nm in enumerate(meta['names']):
        m = meta['regime'] == i
        if not m.any() or m.all():
            continue
        m &= ~bnd  # checked finite above
        sub = [OrderedDict((k, d[k][m]) for k in keys) for d in (got, r32, r64)]
        worst = max(worst, compare64('%s [%s]' % (tag, nm), *sub))
    return worst


# ----------------------------------------------------------------------------------------------------------------
# CPU: the soft-TD oracle is the reference; the generators reach every regime; the reference is float64
# ----------------------------------------------------------------------------------------------------------------
def _soft_fixtures():
    from tests import test_soft_td as ts
    return ts, ts.fixture_names()


@pytest.mark.filterwarnings('ignore:Implicit dimension choice')
@pytest.mark.filterwarnings('ignore:Using a target size')
def test_soft_td_oracle_bit_exact_on_fixtures():
    """fp32, CPU: every stored reference output of tests/golden/soft_td, and the live reference where importable, for a
    unit upstream gradient and the fixtures' mix"""
    from oracle import ref_loader
    ts, names = _soft_fixtures()
    assert names
    live = ref_loader.load() if ref_loader.available() else None
    for name in names:
        case, t, want = ts.load_fixture(name)
        got = ts.run(sto, case, t, 'cpu')
        for k in want:
            assert np.array_equal(got[k], want[k], equal_nan=True), (name, k)
        if live is not None:
            for grad in ('unit', 'mix'):
                a, b = ts.run(sto, case, t, 'cpu', grad), ts.run(live, case, t, 'cpu', grad)
                for k in b:
                    assert np.array_equal(a[k], b[k], equal_nan=True), (name, grad, k)


@pytest.mark.filterwarnings('ignore:Implicit dimension choice')
def test_soft_td_oracle_bit_exact_on_ported_reference_tests():
    ts, _ = _soft_fixtures()
    got, want = ts.ported_body(sto, 'cpu'), ts._stored_port()
    assert set(got) == set(want)
    for k in want:
        assert np.array_equal(got[k], want[k]), k


@pytest.mark.filterwarnings('ignore:Implicit dimension choice')
@pytest.mark.parametrize('name', list(CASES))
def test_reference_fp64(name):
    op, t, p, meta, refs = _case(name)
    if meta['R'] >= 100:
        frac = regime_fractions(meta)
        assert min(frac.values()) >= REGIME_MIN, (name, frac)
    for path, (r32, r64, _, dtypes) in refs.items():
        assert set(r32) == set(r64) == set(dtypes)
        worst = 0.0
        for k, v in r64.items():
            assert dtypes[k] == torch.float64, (name, path, k, dtypes[k])
            a, b = np.asarray(r32[k], np.float64), np.asarray(v, np.float64)
            fin = np.isfinite(b)
            assert np.array_equal(fin, np.isfinite(a)), (name, path, k, 'fp32 oracle non-finite pattern')
            if not fin.any():
                continue
            scale = float(np.abs(b[fin]).max())
            e32 = float(np.abs(a[fin] - b[fin]).max())
            assert e32 <= SANE * scale, (name, path, k, e32, scale)
            worst = max(worst, e32 / (EPS32 * scale) if scale > 0 else 0.0)
        print('\n[fp64 ref] %-36s %-5s max |fp32 oracle - fp64| = %.1f * 2^-24 * scale' % (name, path, worst))


@pytest.mark.filterwarnings('ignore:Implicit dimension choice')
def test_reference_is_float64_inside():
    """the oracles compute in float64 on float64 operands (not fp32 widened at the end): an fp64-only difference shows"""
    for gen, op in ((lambda: gen_dqfd(9090, 64, 4, 3), 'dqfd'), (lambda: gen_mdqn(9091, 64, 4, 0.03), 'mdqn'),
                    (lambda: gen_sql(9092, 64, 4, 3, 0.5), 'sql'), (lambda: gen_qv(9093, 64, 4), 'qv')):
        _, t, p, _ = gen()
        key = 'reward'
        with float64_default():
            x = to64(t)
            a = call(op, 'ref', x, p, 'unit')
            x[key] = x[key] + 1e-12
            b = call(op, 'ref', x, p, 'unit')
        assert a['out_loss'] != b['out_loss'], op


def test_constructed_rows_are_exact():
    """the special rows hold what the comparison rests on"""
    _, t, p, meta = gen_dqfd(9005, 513, 3, 9, cum=True, vg='tensor')
    e = torch.from_numpy(meta['regime'] == meta['names'].index('edge'))
    qsa = t['q'][torch.arange(513), t['action']]
    assert torch.equal((qsa - t['reward'])[e].abs(), torch.full((int(e.sum()), ), CRITERIA['mse'][1]))
    _, t, p, meta = gen_dqfd(9002, 256, 5, 8, crit='l1', vg='tensor', expert='int')
    tie = torch.from_numpy(meta['regime'] == meta['names'].index('tie'))
    x = t['q'] + p['margin']
    x[torch.arange(256), t['action']] = t['q'][torch.arange(256), t['action']]
    top = x[tie].topk(2, 1)[0]
    ties = top[:, 0] == top[:, 1]
    at_act = x[tie][torch.arange(int(tie.sum())), t['action'][tie]] == top[:, 0]
    assert ties.float().mean() > 0.3 and (ties & at_act).any() and (ties & ~at_act).any()
    _, t, p, meta = gen_mdqn(9031, 256, 6, 1 / 256, crit='l1')
    for nm in ('grid', 'edge'):
        m = torch.from_numpy(meta['regime'] == meta['names'].index(nm))
        lp = (t['target_q'] - t['target_q'].max(1, keepdim=True)[0]).gather(1, t['act'].reshape(-1, 1)).reshape(-1)[m]
        assert (lp == -1).any() and (lp < -1).any() and (lp > -1).any(), nm
    _, t, p, meta = gen_mdqn(9036, 1025, 6, -1 / 256)
    m = torch.from_numpy(meta['regime'] == meta['names'].index('grid'))
    lp = (t['target_q'] - t['target_q'].min(1, keepdim=True)[0]).gather(1, t['act'].reshape(-1, 1)).reshape(-1)[m]
    assert (lp == 1).any() and (lp > 1).any()
    m = torch.from_numpy(meta['regime'] == meta['names'].index('tie'))
    top = t['target_q'][m].topk(2, 1)[0]
    assert torch.equal(top[:, 0], top[:, 1])
    m = torch.from_numpy(meta['regime'] == meta['names'].index('peaked'))
    nq = t['next_q'][m].double()
    assert ((nq - nq.max(1, keepdim=True)[0]) / 0.03 < -104).any(1).float().mean() > 0.9  # exp underflows in fp32
    _, t, p, meta = gen_sql(9045, 1024, 3, 9, 1.0)
    m = torch.from_numpy(meta['regime'] == meta['names'].index('inf'))
    nq = t['next_n_q'][m]
    assert (nq == float('inf')).any(1).any() and (nq == float('-inf')).all(1).any()
    assert ((nq == float('inf')).any(1) & (nq == float('-inf')).any(1)).any()
    _, t, p, meta = gen_sql(9063, 1025, 3, 9, 1.0, nan=True, vg='tensor')
    m = torch.from_numpy(meta['regime'] == meta['names'].index('inf'))
    assert torch.isnan(t['next_n_q'][m]).any(1).any()
    for name in ('huge_neg_dqfd_S1024', 'huge_neg_dqfd_S4099', 'huge_neg_dqfd_S65409'):
        mean_tile = float(_case(name)[4]['unit'][1]['out_loss']) * 128
        assert mean_tile < -2.0 ** 37, (name, mean_tile)  # the mean 128-row tile of the loss sum is below -2^37
    for name in ('huge_dqfd_S4099', 'huge_mdqn_S4099', 'huge_sql_S4099', 'huge_qv_S4099'):
        op, t, p, meta = CASES[name]()
        per = _case(name)[4]['unit'][1]['out_per'].reshape(-1)
        R = meta['R']
        tiles = np.add.reduceat(per[:R] * 1.0, np.arange(0, R, 128))
        assert np.abs(tiles).max() > 2.0 ** 36 * 4, name


# ----------------------------------------------------------------------------------------------------------------
# GPU
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.filterwarnings('ignore:Implicit dimension choice')
@pytest.mark.parametrize('name', list(CASES))
def test_td_soft_dqfd_fp64(name):
    op, t, p, meta, refs = _case(name)
    for path in ('unit', 'mix'):
        r32, r64, rec, _ = refs[path]
        for rep in range(2):
            got = call(op, 'gpu', t, p, path)
            compare_case('%s %s #%d' % (name, path, rep), op, t, p, meta, got, r32, r64, rec)
        if name.startswith('huge_'):
            assert np.isfinite(got['out_loss']), name


def _huge_rows(x, g, frac=0.15):
    rows = torch.rand(x.shape[0], generator=g) < frac
    return rows


@pytest.mark.gpu
@pytest.mark.parametrize('S', [1024, 4099, 65409])
def test_large_magnitude_qntd(S):
    """q_nstep_td_error shares grid_sum_fx: tiles above 2^36 on each of the three loss sums"""
    from tests.test_value_td_fp64 import run_gpu as run_gpu_v, run_ref as run_ref_v
    op, t, p, meta = gen_qn(9100 + S % 97, S, 4, 3, vg='tensor')
    g = cases._g(9101)
    h = _huge_rows(t['q'], g)
    t['q'][h, t['action'][h]] += _huge(g, int(h.sum()))
    for path in ('unit', 'mix'):
        r32, r64 = run_ref_v(op, t, p, path)
        got, _ = run_gpu_v(op, t, p, path)
        compare64('qntd huge S%d %s' % (S, path), got, r32, r64)
        assert np.isfinite(got['out_loss'])


def _large_magnitude_other(op, t, p):
    for rep in range(2):
        with float64_default():
            r64 = cases.run_oracle(rl_oracle, op, to64(t), p)
        r32 = cases.run_oracle(rl_oracle, op, t, p)
        import di_engine_b200 as b2
        got = cases.run_api(b2.rl_utils, op, t, p, device=DEV)
        compare64('%s huge #%d' % (op, rep), got, r32, r64)
        for k, v in got.items():
            if k.startswith('out_') and np.asarray(v).ndim == 0:
                assert np.isfinite(v), (op, k)


@pytest.mark.gpu
def test_large_magnitude_a2c():
    """a2c_error's three sums on grid_sum_fx (8 CTAs), value errors ~1e6 in 15 % of the samples"""
    op, t, p = cases.a2c_case(9110, 2000, 6, weight='tensor')
    g = cases._g(9111)
    h = _huge_rows(t['value'], g)
    t['value'][h] += _huge(g, int(h.sum()))
    _large_magnitude_other(op, t, p)


@pytest.mark.gpu
def test_large_magnitude_qrdqn():
    """qrdqn_nstep_td_error on grid_sum_fx (one CTA per sample, 300 CTAs), quantiles ~1e6 in 15 % of the samples"""
    op, t, p, _ = gen_qt(9120, 'qrdqn', 300, 3, 16, 16, 3)
    g = cases._g(9121)
    h = _huge_rows(t['q'], g)
    t['q'][h] += 1e5 * _huge(g, int(h.sum())).reshape(-1, 1, 1)  # one CTA per sample: partial sums of ~1e11 and more
    _large_magnitude_other(op, t, p)


# ---- non-finite operands ------------------------------------------------------------------------------------------
def _poison(t, keys, seed, vals):
    """``vals`` (NaN, +inf, -inf) at a few rows of each operand in ``keys``"""
    g = cases._g(seed)
    t = OrderedDict((k, v.clone() if isinstance(v, torch.Tensor) else v) for k, v in t.items())
    for i, k in enumerate(keys):
        x = t[k]
        R = x.shape[-1] if k == 'reward' and x.dim() == 2 else x.shape[0]
        for val in vals:
            rows = torch.randint(0, R, (3, ), generator=g)
            if k == 'reward' and x.dim() == 2:
                x[0, rows] = val
            elif x.dim() == 1:
                x[rows] = val
            else:
                x[rows, torch.randint(0, x.shape[-1], (3, ), generator=g)] = val
    return t


NONFINITE = [
    ('dqfd', lambda S: gen_dqfd(9130 + S % 97, S, 4, 3, vg='tensor'), ('q', 'next_n_q', 'new_n_q_one_step', 'reward')),
    ('mdqn', lambda S: gen_mdqn(9131 + S % 97, S, 4, 0.03), ('q', 'target_q', 'next_q', 'reward')),
    ('sql', lambda S: gen_sql(9132 + S % 97, S, 4, 3, 0.5), ('q', 'next_n_q', 'reward')),
    ('qv', lambda S: gen_qv(9133 + S % 97, S, 4), ('q', 'v', 'reward')),
]


@pytest.mark.gpu
@pytest.mark.filterwarnings('ignore:Implicit dimension choice')
@pytest.mark.parametrize('S', [1000, 4099, 65409])
@pytest.mark.parametrize('kind,vals', [(k, v) for k, _, _ in NONFINITE for v in ('mixed', 'inf')] + [('dqfd', 'neginf')])
def test_nonfinite_pattern(kind, vals, S):
    """NaN / +-inf in q, target_q, next_q and reward ('mixed'); +inf rewards alone on weighted rows ('inf': the loss is
    +inf, on every row count); +inf one-step next values on live weighted rows with lambda_1 < 0 ('neginf', DQfD: the loss
    and the per-sample errors are -inf, the one-step statistic +inf): every output holds NaN / +inf / -inf exactly where the
    float64 reference does, and the rest is within the bound"""
    gen, keys = next((g, k) for n, g, k in NONFINITE if n == kind)
    op, t, p, meta = gen(S)
    if vals == 'neginf':
        p = dict(p, lam=(1.0, 1.0, -1.5))
        t = OrderedDict((k, v.clone() if isinstance(v, torch.Tensor) else v) for k, v in t.items())
        rows = torch.randint(0, S, (3, ), generator=cases._g(9150 + S))
        t['done_one_step'][rows] = 0.0
        t['weight'][rows] = 1.0
        t['new_n_q_one_step'][rows, t['next_n_action_one_step'][rows]] = float('inf')
    elif vals == 'inf':
        t['weight'] = t['weight'] + 0.25
        t = _poison(t, ('reward', ), 9140 + S, (float('inf'), ))
    else:
        t = _poison(t, keys, 9140 + S, (float('nan'), float('inf'), float('-inf')))
    with float64_default():
        r64 = call(op, 'ref', to64(t), p, 'unit')
    r32 = call(op, 'ref', t, p, 'unit')
    got = call(op, 'gpu', t, p, 'unit')
    for k in r64:
        x, b = np.asarray(got[k]).reshape(-1), np.asarray(r64[k]).reshape(-1)
        nf = ~np.isfinite(b)
        assert np.array_equal(np.isnan(x), np.isnan(b)), (kind, S, k, 'NaN pattern', int((np.isnan(x) != np.isnan(b)).sum()))
        assert np.array_equal(x[nf & ~np.isnan(b)], b[nf & ~np.isnan(b)]), (kind, S, k, 'inf pattern')
    if vals != 'mixed':  # the reference's loss is the infinity the variant is built for
        assert float(r64['out_loss']) == (float('-inf') if vals == 'neginf' else float('inf')), (kind, vals, S)
    fin = OrderedDict((k, v) for k, v in r64.items() if np.isfinite(v).all() and k != 'out_clip')
    compare64('nonfinite %s S%d' % (kind, S), *[OrderedDict((k, d[k]) for k in fin) for d in (got, r32, r64)])


# ---- the workspace cap --------------------------------------------------------------------------------------------
# the 128-thread build keeps K partial sums per CTA below word WS_PARTIAL_LIMIT_WORDS (256000) of the workspace, after 16
# control words: (256000 - 16) // K CTAs of 128 rows
def _cap(K_):
    return (256000 - 16) // K_ * 128


CAP = [('dqfd', 4, lambda S: gen_dqfd(9150, S, 2, 1)), ('mdqn', 2, lambda S: gen_mdqn(9151, S, 2, 0.03)),
       ('qv', 1, lambda S: gen_qv(9152, S, 1))]


@pytest.mark.gpu
@pytest.mark.filterwarnings('ignore:Implicit dimension choice')
@pytest.mark.parametrize('kind', [k for k, _, _ in CAP])
def test_workspace_cap(kind):
    """the largest batch whose partial sums fit the workspace matches the reference; one row more is an error, never a
    silent truncation"""
    from di_engine_b200 import _lib
    K_, gen = next((k, g) for n, k, g in CAP if n == kind)
    S = _cap(K_)
    assert kind != 'dqfd' or S == 8191488
    op, t, p, meta = gen(S + 1)
    with pytest.raises(_lib.B200RLError, match='workspace'):
        call(op, 'gpu', t, p, 'unit')
    t = OrderedDict((k, (v[:S] if k != 'reward' or v.dim() == 1 else v[:, :S]) if isinstance(v, torch.Tensor) and
                     v.dim() > 0 else v) for k, v in t.items())
    got = call(op, 'gpu', t, p, 'unit')
    r32 = call(op, 'ref', t, p, 'unit')
    with float64_default():
        r64 = call(op, 'ref', to64(t), p, 'unit')
    r32.pop('out_clip', None)
    r64.pop('out_clip', None)
    got.pop('out_clip', None)
    compare64('workspace cap %s S%d' % (kind, S), got, r32, r64)
