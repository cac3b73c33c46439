"""The UPGO, continuous V-trace, ACER and Retrace kernels against a float64 reference, on masked, clipped, long-horizon
and non-finite batches.

Kernels: ``upgo_fwd_kernel`` / ``upgo_bwd_kernel`` and ``tbce_fwd_kernel`` / ``tbce_bwd_kernel`` (upgo_loss,
tb_cross_entropy), the UPGO mode of ``lambda_scan_kernel`` and ``lambda_returns_bwd_kernel`` (upgo_returns),
``vtc_rows_kernel`` -> ``vtrace_scan_kernel`` -> ``vtc_bwd_kernel`` (vtrace_error_continuous_action), the ACER heads
(``acer_policy_fwd/bwd``, ``acer_value_fwd/bwd``, ``acer_trust_region_kernel``) and ``retrace_kernel``
(compute_q_retraces).

The seeded parity cases draw tame ``randn`` operands.  The generators below draw each row from several regimes: logits
shifted by +-50, saturated with an improbable taken action, or with the other actions masked by -1e8 / -inf; importance
weights of 0, at most 1 and far above 1; UPGO traces that always continue, always cut, or sit exactly on the
``r_{t+1} + V_{t+2} >= V_{t+1}`` tie; continuous policies with sigma from 1e-3 to 1e2 and log-ratios past fp32's exp
range; ACER ratios of 0, at and beyond ``c`` and 1e6, near-deterministic and uniform log-policies, ``Q - V``
cancellation and trust-region rows on both sides of the ``scale`` clamp and exactly on it; Retrace episode ends and
ratios exactly 1.  Shapes straddle every hand-off of the launch code (thread / warp rows, the capped forward and backward
grids, 8- / 16-column scan tiles and their chunk edges, the ACER grid-stride cap, the Retrace column tiles and chunks).

Reference: ``cases.run_oracle`` on float64 copies of the inputs (every fp32 value is exact in double).  The UPGO trace
indicator is a comparison: the reference on the user's fp32 inputs takes it in fp32, so the float64 reference takes it
from the fp32 operands too (and both sides of the tie are pinned by an exact dyadic regime).  The fp32 oracle on the fp32
inputs is the yardstick: for every output X,

    max|X_gpu - X_64| <= K * max(max|X_32 - X_64|, 2^-24 * scale_X)

over the whole tensor and again over the rows of each regime alone; ``scale_X`` is max|X_64|, or for a signed loss the
float64 mean of its per-sample |term|.  Rows on a branch point of the reference (an ACER ratio equal to ``c``, where the
bias weight is 0 in fp32 and 1e-9 in fp64; ``g.k`` within rounding of ``delta`` in the trust region) are left out of the
elementwise check of the outputs that branch, but must be finite.  Every case runs with the upstream gradients the
forward launch expects and with upstream mixes through the backward launch (zeros included), and backward runs twice
through the same graph.
"""
import contextlib
import functools
import math
from collections import OrderedDict

import numpy as np
import pytest
import torch

from oracle import rl_oracle
from tests import cases
from tests.test_offpolicy_fp64 import EPS32, K, compare64
from tests.test_value_td_fp64 import _regimes, float64_default, to64

assert K == 8.0  # the bound of the PPO-family fp64 suite, shared, not loosened here
DEV = 'cuda'
NUM_SMS = 132
REGIME_MIN = 0.02
SANE = 2.0 ** -12  # the fp32 oracle's own error, relative to the output's scale, that still makes it a yardstick
_np = cases._np


# ----------------------------------------------------------------------------------------------------------------
# the UPGO trace indicator from the fp32 operands
# ----------------------------------------------------------------------------------------------------------------
def _upgo_returns_fp32_indicator(rewards, bootstrap_values):
    """rl_oracle.upgo_returns with ``r_t + V_{t+1} >= V_t`` evaluated on the fp32 operands, whatever the dtype.  The
    same recurrence and roundings as generalized_lambda_returns with gamma 1 and no done (1 - lambda_t == gamma_t -
    trace_t, the factors 1 are exact), on per-step views: autograd through the in-place loop is quadratic in T."""
    keep = (rewards.float() + bootstrap_values[1:].float()) >= bootstrap_values[:-1].float()
    keep = torch.cat([keep[1:], torch.ones_like(keep[-1:])], dim=0).to(rewards.dtype)
    r, nxt, lam = rewards.unbind(0), bootstrap_values[1:].unbind(0), keep.unbind(0)
    T = len(r)
    out = [None] * T
    out[T - 1] = r[T - 1] + nxt[T - 1]
    for t in range(T - 2, -1, -1):
        out[t] = r[t] + (lam[t] * out[t + 1] + (1 - lam[t]) * nxt[t])
    return torch.stack(out, 0)


@contextlib.contextmanager
def fp32_indicator():
    old = rl_oracle.upgo_returns
    rl_oracle.upgo_returns = _upgo_returns_fp32_indicator
    try:
        yield
    finally:
        rl_oracle.upgo_returns = old


# ----------------------------------------------------------------------------------------------------------------
# generators: every row draws one regime per family; meta['fam'] = {family: (regime per row, names)}
# ----------------------------------------------------------------------------------------------------------------
LOGIT_REGIMES = ('plain', 'shift', 'saturated', 'mask1e8', 'maskinf')
RHO_REGIMES = ('rho0', 'rho_le1', 'rho_large')
IND_REGIMES = ('mixed', 'continue', 'cut', 'tie')


def _in(reg, names, nm):
    return reg == names.index(nm)


def _upgo_logits(g, R, Kk, N):
    """R rows of Kk x N logits and actions; the regime is per row (all Kk sub-rows)"""
    reg = _regimes(g, R, LOGIT_REGIMES)
    z = torch.randn(R, Kk, N, generator=g)
    act = torch.randint(0, N, (R, Kk), generator=g)
    m = _in(reg, LOGIT_REGIMES, 'shift')
    z[m] += (torch.rand(R, 1, 1, generator=g) * 100.0 - 50.0)[m]
    m = _in(reg, LOGIT_REGIMES, 'saturated')
    z[m] *= 8.0
    act[m] = z[m].argmin(-1)  # the taken action is the least probable one
    taken = torch.zeros(R, Kk, N, dtype=torch.bool)
    taken.scatter_(-1, act.unsqueeze(-1), True)
    for nm, val in (('mask1e8', -1e8), ('maskinf', -math.inf)):
        m = _in(reg, LOGIT_REGIMES, nm)
        msk = (torch.rand(R, Kk, N, generator=g) < 0.3) & m.view(R, 1, 1)
        msk |= (m & (torch.rand(R, generator=g) < 0.15)).view(R, 1, 1)  # only the taken action left
        msk &= ~taken
        z[msk] = val
    return z, act, reg


def _traces(g, T, B):
    """rewards (T, B), bootstrap values (T+1, B) and the indicator regime per column"""
    col = _regimes(g, B, IND_REGIMES)
    v = torch.randn(T + 1, B, generator=g)
    r = torch.randn(T, B, generator=g)
    step = v[:-1] - v[1:]
    gap = 0.1 + torch.randn(T, B, generator=g).abs()
    for nm, sign in (('continue', 1.0), ('cut', -1.0)):
        m = _in(col, IND_REGIMES, nm)
        r[:, m] = (step + sign * gap)[:, m]
    m = _in(col, IND_REGIMES, 'tie')  # dyadic: r_t + V_{t+1} == V_t exactly in fp32 and fp64
    vd = torch.randint(-64, 64, (T + 1, B), generator=g).float() / 16.0
    v[:, m] = vd[:, m]
    r[:, m] = (vd[:-1] - vd[1:])[:, m]
    return r, v, col.repeat(T)


def gen_upgo(seed, T, B, N, Kk=None, mask=False, op='upgo'):
    g = cases._g(seed)
    R = T * B
    z, act, lreg = _upgo_logits(g, R, Kk or 1, N)
    t = OrderedDict()
    lead = (T, B) if Kk is None else (T, B, Kk)
    t['target_output'] = z.reshape(*lead, N)
    t['action'] = act.reshape(lead)
    rreg = _regimes(g, R, RHO_REGIMES)
    rho = 1.0 - torch.rand(R, generator=g)  # (0, 1]
    rho[_in(rreg, RHO_REGIMES, 'rho0')] = 0.0
    m = _in(rreg, RHO_REGIMES, 'rho_large')
    rho[m] = (10.0 ** (0.5 + 2.5 * torch.rand(R, generator=g)))[m]
    t['rhos'] = rho.reshape(T, B)
    t['rewards'], t['bootstrap_values'], ireg = _traces(g, T, B)
    t['mask'] = None
    if mask:  # fractional masks on half the entries, 0/1 on the other half
        frac = torch.rand(T, B, Kk, generator=g)
        bern = (torch.rand(T, B, Kk, generator=g) < 0.7).float()
        t['mask'] = torch.where(torch.rand(T, B, Kk, generator=g) < 0.5, frac, bern)
    fam = OrderedDict([('logit', (lreg.numpy(), LOGIT_REGIMES)), ('rho', (rreg.numpy(), RHO_REGIMES)),
                       ('trace', (ireg.numpy(), IND_REGIMES))])
    meta = dict(fam=fam, minf=np.isneginf(z.reshape(R, -1).numpy()), N=N, rows=R)
    if op == 'tbce':
        tt = OrderedDict([('logit', t['target_output']), ('label', t['action']), ('mask', t['mask'])])
        fam.pop('rho')
        fam.pop('trace')
        return 'tbce', tt, {}, meta
    return 'upgo', t, {}, meta


def gen_upret(seed, T, B):
    g = cases._g(seed)
    r, v, ireg = _traces(g, T, B)
    t = OrderedDict([('rewards', r), ('bootstrap_values', v)])
    return 'upret', t, {}, dict(fam=OrderedDict([('trace', (ireg.numpy(), IND_REGIMES))]), rows=T * B)


VTC_REGIMES = ('on_policy', 'in_band', 'sigma_range', 'isw_overflow', 'isw_underflow', 'zero_weight')
VTC_PARAMS = dict(gamma=0.99, lambda_=0.95, rho_clip_ratio=0.9, c_clip_ratio=1.1, rho_pg_clip_ratio=1.3)


def gen_vtc(seed, T, B, D):
    """on_policy: behaviour == target (isw exactly 1); in_band: log isw ~ 0.3 randn, on both sides of every clip;
    sigma_range: sigma 10^U(-3, 2), actions 3..6 sigma from the mean; isw_overflow / isw_underflow: lp - lb = +-(100 + 5D),
    past fp32's exp range (isw inf / 0) and inside fp64's; zero_weight: in_band rows of weight 0"""
    g = cases._g(seed)
    R = T * B
    reg = _regimes(g, R, VTC_REGIMES)
    pick = {nm: (reg == i).view(R, 1) for i, nm in enumerate(VTC_REGIMES)}
    mu = torch.randn(R, D, generator=g)
    sg = torch.exp(0.3 * torch.randn(R, D, generator=g))
    sg = torch.where(pick['sigma_range'], 10.0 ** (5.0 * torch.rand(R, D, generator=g) - 3.0), sg)
    far = torch.where(torch.rand(R, D, generator=g) < 0.5, -1.0, 1.0) * (3.0 + 3.0 * torch.rand(R, D, generator=g))
    act = torch.where(pick['sigma_range'], mu + far * sg, mu + sg * torch.randn(R, D, generator=g))
    mu_b = mu + (0.3 / math.sqrt(D)) * sg * torch.randn(R, D, generator=g)
    sg_b = sg * torch.exp((0.1 / math.sqrt(D)) * torch.randn(R, D, generator=g))
    sg_b = torch.where(pick['sigma_range'], sg, sg_b)
    k = math.sqrt(2.0 * (100.0 / D + 5.0))  # per dimension (k sigma)^2 / (2 sigma^2) = 100 / D + 5
    over, under = pick['isw_overflow'], pick['isw_underflow']
    act = torch.where(over, mu, act)
    mu_b = torch.where(over, mu + k * sg, mu_b)
    mu_b = torch.where(under, act, mu_b)
    mu = torch.where(under, act + k * sg, mu)
    sg_b = torch.where(over | under, sg, sg_b)
    on = pick['on_policy']
    mu_b, sg_b = torch.where(on, mu, mu_b), torch.where(on, sg, sg_b)
    w = 0.5 + torch.rand(R, generator=g)
    w[pick['zero_weight'].view(R)] = 0.0
    t = OrderedDict()
    t['mu_target'], t['sigma_target'] = mu.reshape(T, B, D), sg.reshape(T, B, D)
    t['mu_behaviour'], t['sigma_behaviour'] = mu_b.reshape(T, B, D), sg_b.reshape(T, B, D)
    t['action'] = act.reshape(T, B, D)
    t['value'] = torch.randn(T + 1, B, generator=g)
    t['reward'] = torch.rand(T, B, generator=g)
    t['weight'] = w.reshape(T, B)
    return 'vtc', t, dict(VTC_PARAMS), dict(fam=OrderedDict([('policy', (reg.numpy(), VTC_REGIMES))]), rows=R)


RATIO_REGIMES = ('ratio0', 'below_c', 'at_c', 'above_c', 'ratio1e6')
POLICY_REGIMES = ('log_softmax', 'near_deterministic', 'uniform')
QV_REGIMES = ('qv_plain', 'qv_cancel')
TR_REGIMES = ('scale_zero', 'scale_pos', 'scale_edge')


def gen_acer(seed, T, B, N, c=10.0, delta=1.0):
    """ratio: the taken action and ~70 % of the others in the row's regime, the rest U(0, 1.5c); near_deterministic
    log-policies: -1e-7 at one action, -40 elsewhere; qv_cancel: V ~ 100, Q and Qret within 1e-3 of V; trust region:
    g.k well below / above delta, or k = 1 (avg_logit 0) and dyadic g with sum exactly delta"""
    g = cases._g(seed)
    M = T * B
    rr = _regimes(g, M, RATIO_REGIMES)
    pr = _regimes(g, M, POLICY_REGIMES)
    qr = _regimes(g, M, QV_REGIMES)
    tr = _regimes(g, M, TR_REGIMES)
    act = torch.randint(0, N, (M, ), generator=g)
    val = {'ratio0': torch.zeros(M, N), 'below_c': c * (0.05 + 0.9 * torch.rand(M, N, generator=g)),
           'at_c': torch.full((M, N), c), 'above_c': c * (1.05 + 2.0 * torch.rand(M, N, generator=g)),
           'ratio1e6': torch.full((M, N), 1e6)}
    ratio = torch.rand(M, N, generator=g) * 1.5 * c
    own = torch.rand(M, N, generator=g) < 0.7
    own[torch.arange(M), act] = True
    for i, nm in enumerate(RATIO_REGIMES):
        m = (rr == i).view(M, 1) & own
        ratio[m] = val[nm][m]
    logit = torch.log_softmax(torch.randn(M, N, generator=g), -1)
    m = _in(pr, POLICY_REGIMES, 'near_deterministic')
    det = torch.full((M, N), -40.0)
    det[torch.arange(M), torch.randint(0, N, (M, ), generator=g)] = -1e-7
    logit[m] = det[m]
    logit[_in(pr, POLICY_REGIMES, 'uniform')] = -math.log(N)
    q = torch.randn(M, N, generator=g)
    v = torch.randn(M, generator=g)
    qret = torch.randn(M, generator=g)
    m = _in(qr, QV_REGIMES, 'qv_cancel')
    vc = 100.0 + torch.randn(M, generator=g)
    v[m] = vc[m]
    q[m] = (vc.view(M, 1) + 1e-3 * torch.randn(M, N, generator=g))[m]
    qret[m] = (vc + 1e-3 * torch.randn(M, generator=g))[m]
    avg = torch.log_softmax(torch.randn(M, N, generator=g), -1)
    grad = 0.5 * torch.randn(M, N, generator=g)
    m = _in(tr, TR_REGIMES, 'scale_zero')
    grad[m] -= 1.0
    m = _in(tr, TR_REGIMES, 'scale_pos')
    grad[m] += 4.0 * delta
    m = _in(tr, TR_REGIMES, 'scale_edge')
    avg[m] = 0.0
    dy = torch.randint(-32, 32, (M, N), generator=g).float() / 16.0
    dy[:, -1] = delta - dy[:, :-1].sum(-1)
    grad[m] = dy[m]
    w = torch.linspace(0.5, 1.5, M)  # the upstream gradient of each per-transition loss, zeros included
    w[torch.rand(M, generator=g) < 0.05] = 0.0
    t = OrderedDict()
    t['q_values'] = q.reshape(T, B, N)
    t['q_retraces'] = qret.reshape(T, B, 1)
    t['v_pred'] = v.reshape(T, B, 1)
    t['target_logit'] = logit.reshape(T, B, N)
    t['actions'] = act.reshape(T, B)
    t['ratio'] = ratio.reshape(T, B, N)
    t['avg_logit'] = avg.reshape(T, B, N)
    t['actor_gradient'] = grad.reshape(T, B, N)
    t['_w'] = w
    fam = OrderedDict([('ratio', (rr.numpy(), RATIO_REGIMES)), ('policy', (pr.numpy(), POLICY_REGIMES)),
                       ('qv', (qr.numpy(), QV_REGIMES)), ('trust', (tr.numpy(), TR_REGIMES))])
    return 'acer', t, dict(c_clip_ratio=c, trust_region_value=delta), dict(fam=fam, rows=M, N=N)


RT_REGIMES = ('live', 'episode_end', 'ratio_one', 'ratio_below', 'ratio_above')


def gen_retrace(seed, T, B, N, gamma=0.99):
    g = cases._g(seed)
    R = T * B
    reg = _regimes(g, R, RT_REGIMES)
    act = torch.randint(0, N, (R, ), generator=g)
    w = torch.rand(R, generator=g)
    w[_in(reg, RT_REGIMES, 'episode_end')] = 0.0
    ratio = torch.rand(R, N, generator=g) * 0.8 + 0.6
    ra = ratio[torch.arange(R), act]
    ra[_in(reg, RT_REGIMES, 'ratio_one')] = 1.0
    m = _in(reg, RT_REGIMES, 'ratio_below')
    ra[m] = (0.2 + 0.79 * torch.rand(R, generator=g))[m]
    m = _in(reg, RT_REGIMES, 'ratio_above')
    ra[m] = (1.01 + 2.0 * torch.rand(R, generator=g))[m]
    ratio[torch.arange(R), act] = ra
    t = OrderedDict()
    t['q_values'] = torch.randn(T + 1, B, N, generator=g)
    t['v_pred'] = torch.randn(T + 1, B, 1, generator=g)
    t['rewards'] = torch.randn(T, B, generator=g)
    t['actions'] = act.reshape(T, B)
    t['weights'] = w.reshape(T, B)
    t['ratio'] = ratio.reshape(T, B, N)
    return 'retrace', t, dict(gamma=gamma), dict(fam=OrderedDict([('step', (reg.numpy(), RT_REGIMES))]), rows=R)


# ----------------------------------------------------------------------------------------------------------------
# runners: the same code for the oracle (CPU, fp32 or fp64) and the package (GPU); each returns the first backward's
# results and the gradients of a second backward through the same graph
# ----------------------------------------------------------------------------------------------------------------
PATHS = {
    'upgo': ('unit', 'mix'),  # the forward-written unit gradient / 0.7 through the backward launch
    'tbce': ('ones', 'mix'),
    'upret': ('ones', 'mix'),
    'vtc': ('impala', 'policy_only', 'value_only', 'entropy_only'),
    'acer': ('both', 'actor_only', 'bias_only'),
    'retrace': ('forward', ),
}
VTC_MIX = {'impala': [1.0, 0.5, -0.01], 'policy_only': [1.0, 0.0, 0.0], 'value_only': [0.0, 1.0, 0.0],
           'entropy_only': [0.0, 0.0, 1.0]}
GRAD_IN = {'upgo': ['target_output'], 'tbce': ['logit'], 'upret': ['rewards', 'bootstrap_values'],
           'vtc': ['mu_target', 'sigma_target', 'value'], 'acer': ['target_logit', 'q_values'], 'retrace': []}


def _upstream(shape, path, like):
    """an fp32 upstream gradient for a (T, B) output: ones, or randn with 20 % zeros"""
    f32 = torch.float32  # the same draws also under a float64 default dtype
    if path == 'ones':
        x = torch.ones(shape, dtype=f32)
    else:
        g = cases._g(9300 + int(np.prod(shape)))
        x = torch.randn(shape, generator=g, dtype=f32)
        x[torch.rand(shape, generator=g, dtype=f32) < 0.2] = 0.0
    return x.to(dtype=like.dtype, device=like.device)


def _prep(op, t, device):
    out = OrderedDict()
    for k, v in t.items():
        if isinstance(v, torch.Tensor):
            v = v.clone().to(device)
            if k in GRAD_IN[op]:
                v.requires_grad_(True)
        out[k] = v
    return out


def _forward(api, op, tt, p, path):
    """(outputs, the scalar whose gradient is taken)"""
    res = OrderedDict()
    if op == 'upgo':
        loss = api.upgo_loss(tt['target_output'], tt['rhos'], tt['action'], tt['rewards'], tt['bootstrap_values'],
                             tt['mask'])
        res['out_loss'] = _np(loss)
        return res, loss if path == 'unit' else 0.7 * loss
    if op == 'tbce':
        ce = api.tb_cross_entropy(tt['logit'], tt['label'], tt['mask'])
        res['out_ce'] = _np(ce)
        return res, (ce * _upstream(tuple(ce.shape), path, ce)).sum()
    if op == 'upret':
        ret = api.upgo_returns(tt['rewards'], tt['bootstrap_values'])
        res['out_ret'] = _np(ret)
        return res, (ret * _upstream(tuple(ret.shape), path, ret)).sum()
    if op == 'vtc':
        if api is rl_oracle:
            out = rl_oracle.vtrace_error_continuous_action(**tt, **p)
        else:
            data = api.vtrace_data({'mu': tt['mu_target'], 'sigma': tt['sigma_target']},
                                   {'mu': tt['mu_behaviour'], 'sigma': tt['sigma_behaviour']}, tt['action'], tt['value'],
                                   tt['reward'], tt['weight'])
            out = api.vtrace_error_continuous_action(data, **p)
        for k, v in zip(('policy_loss', 'value_loss', 'entropy_loss'), out):
            res['out_' + k] = _np(v)
        return res, sum(c * l for c, l in zip(VTC_MIX[path], out))
    if op == 'acer':
        actor, bias = api.acer_policy_error(tt['q_values'].detach(), tt['q_retraces'], tt['v_pred'], tt['target_logit'],
                                            tt['actions'], tt['ratio'], p['c_clip_ratio'])
        critic = api.acer_value_error(tt['q_values'], tt['q_retraces'], tt['actions'])
        res['out_actor_loss'], res['out_bias_correction_loss'], res['out_critic_loss'] = _np(actor), _np(bias), _np(critic)
        res['out_trust_region'] = _np(api.acer_trust_region_update([tt['actor_gradient']], tt['target_logit'].detach(),
                                                                   tt['avg_logit'], p['trust_region_value'])[0])
        w = tt['_w'].reshape(actor.shape)
        total = (critic * w.flip(0)).sum()
        if path != 'bias_only':
            total = total + (actor * w).sum()
        if path != 'actor_only':
            total = total + 0.3 * (bias * w.flip(1)).sum()
        return res, total
    if op == 'retrace':
        keys = ('q_values', 'v_pred', 'rewards', 'actions', 'weights', 'ratio')
        res['out_q_retraces'] = _np(api.compute_q_retraces(*[tt[k] for k in keys], **p))
        return res, None
    raise KeyError(op)


def run(api, op, t, p, path, device):
    tt = _prep(op, t, device)
    res, total = _forward(api, op, tt, p, path)
    if total is None:
        return res, None
    total.backward(retain_graph=True)
    for k in GRAD_IN[op]:
        res['grad_' + k] = _np(tt[k].grad)
        tt[k].grad = None
    total.backward()
    res2 = OrderedDict(('grad_' + k, _np(tt[k].grad)) for k in GRAD_IN[op])
    return res, res2


def run_ref(op, t, p, path):
    """(fp32 oracle, fp64 oracle), each (results, second-backward gradients)"""
    with fp32_indicator():
        r32 = run(rl_oracle, op, t, p, path, 'cpu')
        with float64_default():
            r64 = run(rl_oracle, op, to64(t), p, path, 'cpu')
    return r32, r64


def run_gpu(op, t, p, path):
    import di_engine_b200 as b2
    return run(b2.rl_utils, op, t, p, path, DEV)


# ----------------------------------------------------------------------------------------------------------------
# loss scales, boundary rows, per-row views
# ----------------------------------------------------------------------------------------------------------------
def scales(op, t, p):
    """float64 mean |term| of each signed loss"""
    t = to64(t)
    if op == 'upgo':
        with torch.no_grad():
            adv = t['rhos'] * (_upgo_returns_fp32_indicator(t['rewards'], t['bootstrap_values']) -
                               t['bootstrap_values'][:-1])
            metric = rl_oracle.tb_cross_entropy(t['target_output'], t['action'], t['mask'])
        return {'out_loss': float((adv * metric).abs().mean())}
    if op == 'vtc':
        def logp(mu, sg):
            return (-((t['action'] - mu) ** 2) / (2 * sg ** 2) - sg.log() - math.log(math.sqrt(2 * math.pi))).sum(-1)

        lp = logp(t['mu_target'], t['sigma_target'])
        isw = torch.exp(lp - logp(t['mu_behaviour'], t['sigma_behaviour']))
        v, r, gm = t['value'], t['reward'], p['gamma']
        deltas = isw.clamp(max=p['rho_clip_ratio']) * (r + gm * v[1:] - v[:-1])
        cs = isw.clamp(max=p['c_clip_ratio'])
        vs, carry = v[:-1].clone(), 0.
        for i in range(r.shape[0] - 1, -1, -1):
            carry = deltas[i] + gm * p['lambda_'] * cs[i] * carry
            vs[i] += carry
        adv = isw.clamp(max=p['rho_pg_clip_ratio']) * (r + gm * torch.cat([vs[1:], v[-1:]], 0) - v[:-1])
        ent = (0.5 + 0.5 * math.log(2 * math.pi) + torch.log(t['sigma_target'])).sum(-1)
        return {'out_policy_loss': float((lp * adv * t['weight']).abs().mean()),
                'out_entropy_loss': float((ent * t['weight']).abs().mean())}
    return {}


def boundary(op, t, p, meta):
    """{output key: rows on a branch point of the fp64 reference}"""
    if op != 'acer':
        return {}
    at_c = (t['ratio'] == np.float32(p['c_clip_ratio'])).reshape(meta['rows'], -1).any(-1).numpy()
    g = t['actor_gradient'].double().reshape(meta['rows'], -1)
    k = torch.exp(t['avg_logit'].double()).reshape(meta['rows'], -1)
    gk, mag = (g * k).sum(-1), (g * k).abs().sum(-1)
    edge = ((gk - p['trust_region_value']).abs() <= 1e-5 * (mag + p['trust_region_value'])).numpy()
    return {'grad_target_logit': at_c, 'out_trust_region': edge}


def rows(op, key, x):
    """``x`` with one entry per regime row on axis 0, or None for a scalar output"""
    x = np.asarray(x)
    if x.ndim == 0:
        return None
    if op == 'vtc' and key == 'grad_value' or op == 'retrace':  # (T+1, B[, 1]): row T is the bootstrap value
        x = x[:-1]
    if op == 'upret' and key == 'grad_bootstrap_values':  # V_{t+1} enters step t; V_0 gets no gradient
        x = x[1:]
    if op in ('upret', 'tbce') and key in ('out_ret', 'out_ce', 'grad_rewards', 'grad_bootstrap_values'):
        return x.reshape(-1)
    T, B = x.shape[:2]
    return x.reshape(T * B, -1)


def _select(op, d, sel, bnd):
    out = OrderedDict()
    for k, x in d.items():
        xr = rows(op, k, x)
        if xr is None:
            continue
        s = sel & ~bnd[k] if k in bnd else sel
        out[k] = xr[s]
    return out


def compare_case(tag, op, meta, got, r32, r64, sc, bnd):
    """the bound on the whole tensors (boundary rows left out) and on the rows of each regime of each family"""
    R = meta['rows']
    for k, m in bnd.items():
        if k in got and m.any():
            assert np.isfinite(rows(op, k, got[k])[m]).all(), (tag, k, 'non-finite at a boundary row')
    everything = np.ones(R, bool)
    whole = []
    for d in (got, r32, r64):
        w = OrderedDict((k, v) for k, v in d.items() if rows(op, k, v) is None)
        w.update(_select(op, d, everything, bnd))
        whole.append(w)
    worst = compare64(tag, *whole, scales=sc)
    for fam, (reg, names) in meta['fam'].items():
        for i, nm in enumerate(names):
            m = reg == i
            if not m.any() or m.all():
                continue
            sub = [_select(op, d, m, bnd) for d in (got, r32, r64)]
            worst = max(worst, compare64('%s [%s]' % (tag, nm), *sub))
    return worst


# ----------------------------------------------------------------------------------------------------------------
# the cases
# ----------------------------------------------------------------------------------------------------------------
UPGO_THREAD_CAP = NUM_SMS * 16 * 128  # forward rows of the capped thread-per-row grid
UPGO_WARP_CAP = NUM_SMS * 16 * 4      # forward rows of the capped warp-per-row grid
ACER_CAP = NUM_SMS * 8 * 256          # rows of one ACER grid-stride pass

CASES = OrderedDict([
    # UPGO head: thread rows (N <= 64) past the forward cap (and so the backward cap, NUM_SMS * 8 * 128 rows); warp rows
    # (N > 64) past the forward and the backward cap (NUM_SMS * 8 * 4 rows); K = 1 and K > 1 with masks
    ('upgo_N64_T64_B4226', lambda: gen_upgo(9001, 64, 4226, 64)),
    ('upgo_N65_T36_B250', lambda: gen_upgo(9002, 36, 250, 65)),
    ('upgo_K3_N65_T20_B100_mask', lambda: gen_upgo(9003, 20, 100, 65, Kk=3, mask=True)),
    ('upgo_K4_N7_T64_B600_mask', lambda: gen_upgo(9004, 64, 600, 7, Kk=4, mask=True)),
    ('upgo_K2_N64_T8_B50', lambda: gen_upgo(9005, 8, 50, 64, Kk=2)),
    ('upgo_N5_T3000_B40', lambda: gen_upgo(9006, 3000, 40, 5)),
    ('tbce_N64_T32_B300', lambda: gen_upgo(9010, 32, 300, 64, op='tbce')),
    ('tbce_N65_T16_B200', lambda: gen_upgo(9011, 16, 200, 65, op='tbce')),
    ('tbce_K3_N65_T16_B100_mask', lambda: gen_upgo(9012, 16, 100, 65, Kk=3, mask=True, op='tbce')),
    ('tbce_K5_N6_T32_B64_mask', lambda: gen_upgo(9013, 32, 64, 6, Kk=5, mask=True, op='tbce')),
    # upgo_returns: 8-column tiles with 128-step chunks below B = 4224 (16 * 2 * 132 SMs), 16-column tiles with
    # 64-step chunks from there; T = 1, both chunk edges, thousands of steps (the backward's forward chain)
    ('upret_T1_B4223', lambda: gen_upret(9020, 1, 4223)),
    ('upret_T1_B4224', lambda: gen_upret(9021, 1, 4224)),
    ('upret_T63_B4224', lambda: gen_upret(9022, 63, 4224)),
    ('upret_T64_B4224', lambda: gen_upret(9023, 64, 4224)),
    ('upret_T65_B4224', lambda: gen_upret(9024, 65, 4224)),
    ('upret_T64_B4223', lambda: gen_upret(9025, 64, 4223)),
    ('upret_T127_B4223', lambda: gen_upret(9026, 127, 4223)),
    ('upret_T128_B4223', lambda: gen_upret(9027, 128, 4223)),
    ('upret_T129_B4223', lambda: gen_upret(9028, 129, 4223)),
    ('upret_T129_B4224', lambda: gen_upret(9029, 129, 4224)),
    ('upret_T4096_B4223', lambda: gen_upret(9030, 4096, 4223)),
    ('upret_T4096_B4224', lambda: gen_upret(9031, 4096, 4224)),
    # continuous V-trace: the scan's 8- / 16-column tiles at B = 4223 / 4224, T = 64 / 65, long narrow batches
    ('vtc_T64_B4223_D1', lambda: gen_vtc(9040, 64, 4223, 1)),
    ('vtc_T65_B4224_D6', lambda: gen_vtc(9041, 65, 4224, 6)),
    ('vtc_T65_B4223_D17', lambda: gen_vtc(9042, 65, 4223, 17)),
    ('vtc_T64_B4224_D17', lambda: gen_vtc(9043, 64, 4224, 17)),
    ('vtc_T8192_B1_D6', lambda: gen_vtc(9044, 8192, 1, 6)),
    ('vtc_T4096_B7_D1', lambda: gen_vtc(9045, 4096, 7, 1)),
    # ACER: past one grid-stride pass (NUM_SMS * 8 * 256 rows); N = 1, 6, 18, 300; c = 10 and 2
    ('acer_M275200_N6', lambda: gen_acer(9060, 64, 4300, 6)),
    ('acer_M4096_N1', lambda: gen_acer(9061, 32, 128, 1)),
    ('acer_M8192_N18_c2', lambda: gen_acer(9062, 64, 128, 18, c=2.0, delta=0.5)),
    ('acer_M600_N300', lambda: gen_acer(9063, 12, 50, 300)),
    # Retrace: 32-column tiles (B = 31 / 32 / 33 / 4097), 64-step chunks (T = 63 / 64 / 65 / 1000), N = 1 and 300
    ('retrace_T63_B31_N6', lambda: gen_retrace(9080, 63, 31, 6)),
    ('retrace_T64_B32_N1', lambda: gen_retrace(9081, 64, 32, 1)),
    ('retrace_T65_B33_N300', lambda: gen_retrace(9082, 65, 33, 300)),
    ('retrace_T1000_B4097_N4', lambda: gen_retrace(9083, 1000, 4097, 4)),
    ('retrace_T65_B4097_N1', lambda: gen_retrace(9084, 65, 4097, 1, gamma=0.9)),
])


@functools.lru_cache(maxsize=2)
def _case(name):
    op, t, p, meta = CASES[name]()
    refs = {path: run_ref(op, t, p, path) for path in PATHS[op]}
    return op, t, p, meta, scales(op, t, p), boundary(op, t, p, meta), refs


def regime_fractions(meta):
    return {nm: float(np.mean(reg == i)) for reg, names in meta['fam'].values() for i, nm in enumerate(names)}


# ----------------------------------------------------------------------------------------------------------------
# exact checks
# ----------------------------------------------------------------------------------------------------------------
def exact_checks(tag, op, t, p, meta, got):
    if op in ('upgo', 'tbce'):
        key = 'grad_target_output' if op == 'upgo' else 'grad_logit'
        gz = np.asarray(got[key]).reshape(meta['rows'], -1)
        assert np.all(gz[meta['minf']] == 0.0), (tag, 'gradient at a -inf logit')
        if op == 'upgo':
            N = meta['N']
            sub = gz.reshape(-1, N).astype(np.float64)
            tol = 4 * N * EPS32 * np.abs(sub).max()
            assert np.all(np.abs(sub.sum(-1)) <= tol), (tag, 'row sum of the gradient', float(np.abs(sub.sum(-1)).max()))
    if op == 'acer':
        M, N = meta['rows'], meta['N']
        act = t['actions'].reshape(M).numpy()
        off = np.ones((M, N), bool)
        off[np.arange(M), act] = False
        gq = np.asarray(got['grad_q_values']).reshape(M, N)
        assert np.all(gq[off] == 0.0), (tag, 'value gradient off the taken action')
        ratio = t['ratio'].reshape(M, N)
        w32 = (1.0 - p['c_clip_ratio'] / (ratio + 1e-8)).clamp(min=0.0).numpy()
        gl = np.asarray(got['grad_target_logit']).reshape(M, N)
        zero = off & ((w32 == 0.0) | tag.endswith('actor_only'))
        assert np.all(gl[zero] == 0.0), (tag, 'policy gradient off the taken action with bias weight 0')
        g = t['actor_gradient'].reshape(M, N).double().numpy()
        k = np.exp(t['avg_logit'].reshape(M, N).double().numpy())
        out = np.asarray(got['out_trust_region'], np.float64).reshape(M, N)
        delta = p['trust_region_value']
        scale = ((g * k).sum(-1) - delta) / (k * k).sum(-1)
        edge = boundary(op, t, p, meta)['out_trust_region']
        pos = (scale > 0) & ~edge
        err = np.abs((k * out).sum(-1) - delta)
        tol = 8 * EPS32 * ((np.abs(g * k)).sum(-1) + scale * (k * k).sum(-1))
        assert np.all(err[pos] <= tol[pos]), (tag, 'k . out != delta', float((err[pos] / tol[pos]).max()))
        tre = _in(meta['fam']['trust'][0], TR_REGIMES, 'scale_edge')
        assert np.array_equal(out[tre], g[tre]), (tag, 'g . k == delta exactly: scale is 0 and out is g')
    if op == 'vtc':
        assert np.all(np.asarray(got['grad_value'])[-1] == 0.0), (tag, 'gradient of the bootstrap value V_T')


def _keys(d, pre):
    return OrderedDict((k, v) for k, v in d.items() if k.startswith(pre))


# ----------------------------------------------------------------------------------------------------------------
# CPU: the generators reach every regime, the reference is float64, the fp32 oracle is a sane yardstick
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', list(CASES))
def test_reference_fp64(name):
    op, t, p, meta, sc, bnd, refs = _case(name)
    frac = regime_fractions(meta)
    assert min(frac.values()) >= REGIME_MIN, (name, frac)
    for path, ((r32, s32), (r64, s64)) in refs.items():
        assert set(r32) == set(r64)
        worst = 0.0
        for k in r64:
            for d in (r64, s64 or {}):
                if k in d:
                    assert np.asarray(d[k]).dtype == np.float64, (name, path, k, np.asarray(d[k]).dtype)
            a, b = np.asarray(r32[k], np.float64), np.asarray(r64[k], np.float64)
            fin = np.isfinite(b)
            assert np.array_equal(fin, np.isfinite(a)), (name, path, k, 'fp32 oracle non-finite pattern')
            if not fin.any():
                continue
            scale = float(sc.get(k, np.abs(b[fin]).max()))
            e32 = float(np.abs(a[fin] - b[fin]).max())
            assert e32 <= SANE * scale, (name, path, k, e32, scale)
            worst = max(worst, e32 / (EPS32 * scale) if scale > 0 else 0.0)
        print('\n[fp64 ref] %-30s %-12s max |fp32 oracle - fp64| = %.1f * 2^-24 * scale' % (name, path, worst))


def test_regime_checks_are_real():
    """the constructed rows really are what the regimes claim, bit for bit"""
    # exact UPGO ties: r_t + V_{t+1} == V_t in fp32 and in fp64 on every step of a tie column
    op, t, p, meta = gen_upgo(9006, 3000, 40, 5)
    r, v = t['rewards'], t['bootstrap_values']
    tie = torch.from_numpy(_in(meta['fam']['trace'][0], IND_REGIMES, 'tie').reshape(3000, 40)[0])
    assert tie.any()
    assert torch.equal((r + v[1:])[:, tie], v[:-1][:, tie])
    assert torch.equal((r.double() + v[1:].double())[:, tie], v[:-1].double()[:, tie])
    cont = torch.from_numpy(_in(meta['fam']['trace'][0], IND_REGIMES, 'continue').reshape(3000, 40)[0])
    cut = torch.from_numpy(_in(meta['fam']['trace'][0], IND_REGIMES, 'cut').reshape(3000, 40)[0])
    assert bool(((r + v[1:]) >= v[:-1])[:, cont].all()) and bool(((r + v[1:]) < v[:-1])[:, cut].all())
    # ACER: ratios exactly c; trust-region edge rows with g . k == delta exactly in fp32
    op, t, p, meta = gen_acer(9062, 64, 128, 18, c=2.0, delta=0.5)
    M = meta['rows']
    at_c = torch.from_numpy(_in(meta['fam']['ratio'][0], RATIO_REGIMES, 'at_c'))
    taken = t['ratio'].reshape(M, -1)[torch.arange(M), t['actions'].reshape(M)]
    assert torch.all(taken[at_c] == 2.0)
    edge = torch.from_numpy(_in(meta['fam']['trust'][0], TR_REGIMES, 'scale_edge'))
    k = torch.exp(t['avg_logit'].reshape(M, -1)[edge])
    assert torch.all(k == 1.0)
    assert torch.all((t['actor_gradient'].reshape(M, -1)[edge] * k).sum(-1) == 0.5)
    assert bool(boundary(op, t, p, meta)['out_trust_region'][edge.numpy()].all())
    # continuous V-trace: the importance weight overflows / underflows fp32 (and not fp64) on those rows
    op, t, p, meta = gen_vtc(9040, 64, 4223, 1)
    reg = meta['fam']['policy'][0]

    def logp(mu, sg, a):
        return (-((a - mu) ** 2) / (2 * sg ** 2) - sg.log() - math.log(math.sqrt(2 * math.pi))).sum(-1).reshape(-1)

    for dt in (torch.float32, torch.float64):
        tt = {k: v.to(dt) for k, v in t.items()}
        isw = torch.exp(logp(tt['mu_target'], tt['sigma_target'], tt['action']) -
                        logp(tt['mu_behaviour'], tt['sigma_behaviour'], tt['action']))
        over = torch.from_numpy(_in(reg, VTC_REGIMES, 'isw_overflow'))
        under = torch.from_numpy(_in(reg, VTC_REGIMES, 'isw_underflow'))
        on = torch.from_numpy(_in(reg, VTC_REGIMES, 'on_policy'))
        if dt == torch.float32:
            assert torch.isinf(isw[over]).all() and (isw[under] == 0).all()
        else:
            assert torch.isfinite(isw[over]).all() and (isw[under] > 0).all()
        assert (isw[on] == 1.0).all()
    # Retrace: ratios exactly 1 at the taken action
    op, t, p, meta = gen_retrace(9080, 63, 31, 6)
    R = meta['rows']
    one = torch.from_numpy(_in(meta['fam']['step'][0], RT_REGIMES, 'ratio_one'))
    assert torch.all(t['ratio'].reshape(R, -1)[torch.arange(R), t['actions'].reshape(R)][one] == 1.0)


# ----------------------------------------------------------------------------------------------------------------
# GPU
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('name', list(CASES))
def test_actor_critic_fp64(name):
    op, t, p, meta, sc, bnd, refs = _case(name)
    worst = 0.0
    for path in PATHS[op]:
        got, got2 = run_gpu(op, t, p, path)
        (r32, s32), (r64, s64) = refs[path]
        tag = '%s %s' % (name, path)
        worst = max(worst, compare_case(tag, op, meta, got, r32, r64, sc, bnd))
        if got2 is not None:
            worst = max(worst, compare_case(tag + ' 2nd-backward', op, meta, got2, s32, s64, {}, bnd))
        exact_checks(tag, op, t, p, meta, got)
        if op == 'retrace':
            a, b = np.asarray(got['out_q_retraces']), np.asarray(r32['out_q_retraces'])
            assert np.array_equal(a, b, equal_nan=True), (tag, 'not bit-exact with the fp32 oracle')
    print('\n[fp64 worst] %-30s max err_gpu/bound_floor %.2f' % (name, worst))


def _nonfinite_case(kind):
    what, where, v = kind.split('_')
    val = {'nan': math.nan, 'posinf': math.inf, 'neginf': -math.inf}[v]
    if what == 'acer':
        op, t, p, meta = gen_acer(9501, 5, 8, 6)
        key = {'ratio': 'ratio', 'q': 'q_values', 'grad': 'actor_gradient'}[where]
        x = t[key].reshape(40, 6)
        act = t['actions'].reshape(40)
        x[3, act[3]] = val           # at the taken action
        x[11, (act[11] + 1) % 6] = val  # at another action
        x[27, :] = val               # a whole row
        return op, t, p, meta
    if what == 'retrace':
        op, t, p, meta = gen_retrace(9502, 40, 9, 4)
        x = t['ratio'].reshape(360, 4)
        act = t['actions'].reshape(360)
        for r in (7 * 9 + 2, 33 * 9 + 5):
            x[r, act[r]] = val
        return op, t, p, meta
    op, t, p, meta = gen_upgo(9503, 6, 16, 7, op='tbce' if what == 'tbce' else 'upgo')
    if where == 'rhos':
        t['rhos'][2, 5] = val
    else:
        z = t['logit' if what == 'tbce' else 'target_output']
        z[1, 3, 2] = val
        z[4, 9, :2] = val
    return op, t, p, meta


NONFINITE = ['acer_ratio_nan', 'acer_ratio_posinf', 'acer_ratio_neginf', 'acer_q_nan', 'acer_q_posinf', 'acer_q_neginf',
             'acer_grad_nan', 'acer_grad_posinf', 'acer_grad_neginf', 'retrace_ratio_nan', 'upgo_rhos_nan',
             'upgo_logit_posinf', 'tbce_logit_posinf']


@pytest.mark.gpu
@pytest.mark.parametrize('kind', NONFINITE)
def test_nonfinite_operands(kind):
    """NaN and +-inf operands: every output's NaN / +inf / -inf pattern is the fp64 reference's"""
    op, t, p, meta = _nonfinite_case(kind)
    for path in PATHS[op]:
        (r32, s32), (r64, s64) = run_ref(op, t, p, path)
        got, got2 = run_gpu(op, t, p, path)
        tag = '%s %s' % (kind, path)
        for a, b in ((got, r64), (got2 or {}, s64 or {})):
            for k in b:
                x, y = np.asarray(a[k], np.float64), np.asarray(b[k], np.float64)
                for f in (np.isnan, np.isposinf, np.isneginf):
                    assert np.array_equal(f(x), f(y)), (tag, k, f.__name__, int(f(x).sum()), int(f(y).sum()))
        compare64(tag, got, r32, r64)
        if op == 'retrace':
            assert np.array_equal(got['out_q_retraces'], r32['out_q_retraces'], equal_nan=True), tag
