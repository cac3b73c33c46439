"""The value-based TD kernels against a float64 reference, on batches that reach every branch of the target and the loss.

Kernels: ``qntd_fwd_kernel`` / ``qntd_bwd_kernel`` (q_nstep_td_error, _with_rescale, bdq_nstep_td_error, the multi-agent
branch, the R2D2 sequence form and the 1-step / state-value siblings), ``dntd_fwd_kernel`` / ``dntd_bwd_kernel`` (C51:
dist_nstep_td_error, dist_1step_td_error), ``quantile_td_kernel`` (QR-DQN, IQN, FQF) and the TD(lambda) head of
``lambda_scan_kernel``.

The seeded parity cases draw C51 distributions as softmax(randn) (every atom near 1 / n_atom), quantiles as randn (no tie,
no |u| on kappa), Bernoulli ``done`` and uniform rewards.  The generators below draw each row from several regimes:
terminal, fractional and non-binary ``done``; rows placed exactly on a criterion threshold or a Huber edge; exact quantile
ties; peaked, near-converged and subnormal C51 rows; targets that clamp every atom or land on integer bins; reversed
target order (negative ``done`` or ``value_gamma``).  Shapes straddle every geometry hand-off of the kernels (one CTA /
one-round-trip grid sum / ticketed grid sum, 8- / 16-column scan tiles, 2 / 8 atoms per lane, the n-step tail loop past
8 rewards, the 2048-quantile shared-memory cap).

Reference: ``cases.run_oracle`` on float64 copies of the inputs, with float64 as torch's default dtype (the oracle builds
its discount vector and the C51 support in the default dtype).  The fp32 oracle on the fp32 inputs is the yardstick: for
every output X,

    max|X_gpu - X_64| <= K * max(max|X_32 - X_64|, 2^-24 * scale_X)

over the whole tensor, and again over the rows of each regime alone, so that an error on the small outputs of one regime
(a near-converged C51 row has a TD error of 1e-6..1e-3) is not hidden by the larger rows of another.  Each case runs twice:
with a unit upstream gradient (the gradient the forward launch writes) and with an upstream mix through the backward
launch that includes a gradient arriving through the per-sample error.
"""
import contextlib
import functools
from collections import OrderedDict

import numpy as np
import pytest
import torch
import torch.nn as nn

from oracle import rl_oracle
from tests import cases
from tests.test_offpolicy_fp64 import EPS32, K, compare64

assert K == 8.0  # the bound of the PPO-family fp64 suite, shared, not loosened here
DEV = 'cuda'
MIX_LOSS = 0.7  # upstream gradient of the loss in the backward-launch run
REGIME_MIN = 0.02
SANE = 2.0 ** -12  # the fp32 oracle's own error, relative to the output's scale, that still makes it a yardstick


# ----------------------------------------------------------------------------------------------------------------
# helpers
# ----------------------------------------------------------------------------------------------------------------
@contextlib.contextmanager
def float64_default():
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        yield
    finally:
        torch.set_default_dtype(old)


def to64(t):
    return OrderedDict((k, v.double() if isinstance(v, torch.Tensor) and v.is_floating_point() else v)
                       for k, v in t.items())


def _regimes(g, R, names):
    """each row's regime: every regime on an equal share of the rows, in a random order"""
    idx = torch.arange(R) % len(names)
    return idx[torch.randperm(R, generator=g)]


def _zeros_at(g, x, p):
    x = x.clone()
    x[torch.rand(x.shape, generator=g) < p] = 0.0
    return x


def _dyadic(g, n, lo=-64, hi=64, q=16.0):
    return torch.randint(lo, hi, (n, ), generator=g).float() / q


def _per_upstream(shape):
    """the gradient that arrives through the per-sample error in the backward-launch run (zeros included)"""
    g = cases._g(9100 + int(np.prod(shape)))
    x = torch.randn(shape, generator=g, dtype=torch.float32)  # float32 draws also under a float64 default dtype
    x[torch.rand(shape, generator=g, dtype=torch.float32) < 0.2] = 0.0
    return x


class _PerSampleUpstream(torch.autograd.Function):
    """returns ``loss`` unchanged; its backward also sends ``_per_upstream(per.shape)`` into ``per``"""

    @staticmethod
    def forward(ctx, loss, per):
        ctx.like = (per.shape, per.dtype, per.device)
        return loss.clone()

    @staticmethod
    def backward(ctx, g):
        shape, dtype, device = ctx.like
        return g, _per_upstream(shape).to(dtype=dtype, device=device)


LOSS_FNS = {  # public loss function -> index of its differentiable per-sample output
    'q_nstep_td_error': 1, 'q_nstep_td_error_with_rescale': 1, 'bdq_nstep_td_error': 1, 'q_nstep_td_error_sequence': 2,
    'q_1step_td_error': None, 'v_1step_td_error': 1, 'v_nstep_td_error': 1, 'dist_nstep_td_error': 1,
    'dist_1step_td_error': None, 'qrdqn_nstep_td_error': 1, 'iqn_nstep_td_error': 1, 'fqf_nstep_td_error': 1,
    'td_lambda_error': None,
}


class _Api:
    """``api`` (the package's rl_utils or the oracle) with its loss functions wrapped: ``per_grad`` routes an upstream
    gradient into the per-sample error; ``stash`` keeps what the C51 forward saved (its projection)."""

    def __init__(self, api, per_grad):
        self.api, self.per_grad, self.stash = api, per_grad, {}

    def __getattr__(self, name):
        fn = getattr(self.api, name)
        if name not in LOSS_FNS:
            return fn

        def wrapped(*a, **kw):
            out = fn(*a, **kw)
            loss = out[0] if isinstance(out, tuple) else out
            node = loss.grad_fn
            if name == 'dist_nstep_td_error' and node is not None and type(node).__name__.startswith('DistNStep'):
                self.stash['proj'] = node.saved_tensors[2].detach().cpu().numpy().astype(np.float64)
            i = LOSS_FNS[name]
            if self.per_grad and i is not None:
                out = (_PerSampleUpstream.apply(out[0], out[i]), ) + tuple(out[1:])
            return out

        return wrapped


@contextlib.contextmanager
def _mix(op, mix):
    old = cases.LOSS_MIX[op]
    cases.LOSS_MIX[op] = list(mix)
    try:
        yield
    finally:
        cases.LOSS_MIX[op] = old


PATHS = {'unit': ([1.0], False), 'mix': ([MIX_LOSS], True)}


def run_ref(op, t, p, path):
    """(fp32 oracle, fp64 oracle) results for one upstream path"""
    mix, per = PATHS[path]
    with _mix(op, mix):
        r32 = cases.run_oracle(_Api(rl_oracle, per), op, t, p)
        with float64_default():
            r64 = cases.run_oracle(_Api(rl_oracle, per), op, to64(t), p)
    return r32, r64


def run_gpu(op, t, p, path):
    import di_engine_b200 as b2
    mix, per = PATHS[path]
    api = _Api(b2.rl_utils, per)
    with _mix(op, mix):
        res = cases.run_api(api, op, t, p, device=DEV)
    return res, api.stash


# ----------------------------------------------------------------------------------------------------------------
# q-n-step family (qntd_fwd_kernel): terminal / fractional / non-binary done, rows on the criterion threshold
# ----------------------------------------------------------------------------------------------------------------
CRITERIA = {
    'mse': (lambda: nn.MSELoss(reduction='none'), 0.75),  # (module, |d| of the threshold rows)
    'l1': (lambda: nn.L1Loss(reduction='none'), 0.0),
    'smoothl1': (lambda: nn.SmoothL1Loss(reduction='none', beta=2.0), 2.0),
    'huber': (lambda: nn.HuberLoss(reduction='none', delta=0.5), 0.5),
}
QN_REGIMES = ('live', 'terminal', 'fractional', 'nonbinary', 'threshold')
QN_REGIMES_RESCALE = ('live', 'terminal', 'fractional', 'nonbinary')


def _qn_done(g, reg, names):
    S = reg.shape[0]
    done = torch.zeros(S)
    pick = {n: reg == i for i, n in enumerate(names)}
    done[pick['terminal']] = 1.0
    done[pick['fractional']] = torch.rand(S, generator=g)[pick['fractional']]
    done[pick['nonbinary']] = (3.0 * torch.randn(S, generator=g))[pick['nonbinary']]
    if 'threshold' in pick:
        done[pick['threshold']] = 1.0
    return done, pick


def _value_gamma(g, kind, S, t, p, neg=False):
    if kind == 'tensor':
        vg = torch.rand(S, generator=g) * 0.2 + 0.8
        if neg:
            vg[torch.rand(S, generator=g) < 0.1] *= -1.0
        t['value_gamma'] = vg
    elif kind == '0dim':
        t['value_gamma'] = torch.tensor(0.9)
    elif kind == 'float':
        p['value_gamma'] = 0.857


def gen_qn(seed, S, N, nstep, crit='mse', vg=None, weight=True, rescale=False, G=None, marl=False):
    """q-n-step operands; the row regimes are per sample.  ``G``: bdq branches (q (S, G, N)); ``marl``: the reference's
    multi-agent branch (q (S, 3, N), action (S, 3, 1)).  Threshold rows: done 1 and one non-zero reward, so the target is
    the dyadic reward r0 exactly, and q_sa = r0 +- the criterion's threshold (dyadic)."""
    g = cases._g(seed)
    names = QN_REGIMES_RESCALE if rescale else QN_REGIMES
    reg = _regimes(g, S, names)
    done, pick = _qn_done(g, reg, names)
    lead = (S, ) if G is None and not marl else (S, G or 3)
    t = OrderedDict()
    t['q'] = torch.randn(*lead, N, generator=g)
    if rescale:  # h^-1 of the next value from 1e-3 to ~1e5
        mag = 10.0 ** (torch.rand(*lead, N, generator=g) * 6.1 - 3.0)
        t['next_n_q'] = torch.where(torch.rand(*lead, N, generator=g) < 0.5, -mag, mag)
    else:
        t['next_n_q'] = torch.randn(*lead, N, generator=g)
    t['action'] = torch.randint(0, N, lead, generator=g)
    t['next_n_action'] = torch.randint(0, N, lead, generator=g)
    reward = torch.rand(nstep, S, generator=g) * 2.0 - 1.0
    if 'threshold' in pick:
        th = pick['threshold']
        r0 = _dyadic(g, S)
        reward[:, th] = 0.0
        reward[0, th] = r0[th]
        sign = torch.where(torch.rand(S, generator=g) < 0.5, -1.0, 1.0)
        qsa = r0 + sign * CRITERIA[crit][1]
        qv = t['q'].reshape(S, -1, N)
        av = t['action'].reshape(S, -1)
        for j in range(qv.shape[1]):
            qv[th, j, av[th, j]] = qsa[th]
    t['reward'] = reward
    t['done'] = done
    t['weight'] = _zeros_at(g, torch.rand(S, generator=g), 0.05) if weight else None
    p = dict(gamma=0.99, nstep=nstep)
    _value_gamma(g, vg, S, t, p)
    if marl:
        t['action'] = t['action'].unsqueeze(-1)
    if G is not None:
        p['cum_reward'] = False
        return 'bdq', t, p, dict(regime=reg.numpy(), names=names)
    if rescale:
        if crit != 'mse':
            p['criterion'] = CRITERIA[crit][0]()
        return 'qntd_rescale', t, p, dict(regime=reg.numpy(), names=names)
    p['cum_reward'] = False
    p['criterion'] = CRITERIA[crit][0]()
    return 'qntd', t, p, dict(regime=reg.numpy(), names=names, crit=crit)


def gen_qseq(seed, T, B, N, nstep, rescale):
    """the R2D2 sequence form: q (T, B, N), reward (T, nstep, B), done / weight / value_gamma (T, B); regimes per (t, b)"""
    g = cases._g(seed)
    S = T * B
    names = QN_REGIMES_RESCALE
    reg = _regimes(g, S, names)
    done, _ = _qn_done(g, reg, names)
    t = OrderedDict()
    t['q'] = torch.randn(T, B, N, generator=g)
    t['next_n_q'] = torch.randn(T, B, N, generator=g) * (30.0 if rescale else 1.0)
    t['action'] = torch.randint(0, N, (T, B), generator=g)
    t['next_n_action'] = torch.randint(0, N, (T, B), generator=g)
    t['reward'] = torch.rand(T, nstep, B, generator=g) * 2.0 - 1.0
    t['done'] = done.reshape(T, B)
    t['weight'] = _zeros_at(g, torch.rand(T, B, generator=g), 0.05)
    t['value_gamma'] = torch.rand(T, B, generator=g) * 0.2 + 0.8
    return 'qseq', t, dict(gamma=0.997, nstep=nstep, rescale=rescale), dict(regime=reg.numpy(), names=names)


def gen_sibling(seed, op, S, N=None, nstep=1):
    """q_1step_td_error / v_1step_td_error / v_nstep_td_error rows (the n = 1 and state-value cases of the same kernel)"""
    g = cases._g(seed)
    names = QN_REGIMES_RESCALE
    reg = _regimes(g, S, names)
    done, _ = _qn_done(g, reg, names)
    t = OrderedDict()
    w = _zeros_at(g, torch.rand(S, generator=g), 0.05)
    if op == 'q1td':
        t['q'] = torch.randn(S, N, generator=g)
        t['next_q'] = torch.randn(S, N, generator=g)
        t['act'] = torch.randint(0, N, (S, ), generator=g)
        t['next_act'] = torch.randint(0, N, (S, ), generator=g)
        t['reward'] = torch.rand(S, generator=g) * 2.0 - 1.0
        t['done'] = done
        t['weight'] = w
        p = dict(gamma=0.99)
    elif op == 'v1td':
        t['v'] = torch.randn(S, generator=g)
        t['next_v'] = torch.randn(S, generator=g)
        t['reward'] = torch.rand(S, generator=g) * 2.0 - 1.0
        t['done'] = done
        t['weight'] = w
        p = dict(gamma=0.99)
    else:
        t['v'] = torch.randn(S, generator=g)
        t['next_n_v'] = torch.randn(S, generator=g)
        t['reward'] = torch.rand(nstep, S, generator=g) * 2.0 - 1.0
        t['done'] = done
        t['weight'] = w
        t['value_gamma'] = torch.rand(S, generator=g) * 0.2 + 0.8
        p = dict(gamma=0.99, nstep=nstep)
    return op, t, p, dict(regime=reg.numpy(), names=names)


# ----------------------------------------------------------------------------------------------------------------
# C51 (dntd_fwd_kernel)
# ----------------------------------------------------------------------------------------------------------------
DN_REGIMES = ('uniform', 'peaked', 'converged', 'subnormal', 'clamped', 'int_bins', 'reversed')
SUBNORMALS = torch.tensor([1e-39, 2.5e-42, 1.4e-45])


def _vrange(n_atom, kind):
    if kind == 'c51':
        return -10.0, 10.0
    h = (n_atom - 1) * 0.125  # delta_z = 0.25: every atom and every bin position is exact
    return -h, h


def gen_dn(seed, B, N, n_atom, nstep, A=None, vrange='dyadic', vg=None, weight='tensor', one_step=False, zeros=False):
    """C51 operands, regimes per batch entry b (the rows of a multi-agent entry share its reward and done):
    uniform  near-uniform dist, Bernoulli done;
    peaked   dist = softmax(8 randn) + 1e-6, as DistributionHead builds it;
    converged  done 1, target one atom k (integer bin: all mass on k), chosen dist[k] = 1 - 10^U(-6, -3);
    subnormal  as converged, the chosen dist row a raw softmax with subnormal entries at atoms of zero projected mass;
    clamped  |reward| 1e3: every atom clamps to v_min or v_max;
    int_bins done 1, reward on an atom: every bin position an integer;
    reversed done from 3 randn (and negative value_gamma entries): (1 - done) * gamma^n < 0 reverses the order of Tz.
    ``zeros`` (dist_1step_td_error only): a further regime with exact zeros in the chosen dist row."""
    g = cases._g(seed)
    names = DN_REGIMES + (('zeros', ) if zeros else ())
    reg = _regimes(g, B, names)
    pick = {n: reg == i for i, n in enumerate(names)}
    Aa = 1 if A is None else A
    R = B * Aa
    v_min, v_max = _vrange(n_atom, vrange)
    support = torch.linspace(v_min, v_max, n_atom)
    dist = torch.softmax(torch.randn(R, N, n_atom, generator=g), -1)
    ndist = torch.softmax(torch.randn(R, N, n_atom, generator=g) * 2.0, -1)
    act = torch.randint(0, N, (R, ), generator=g)
    nact = torch.randint(0, N, (R, ), generator=g)
    reward = torch.randn(nstep, B, generator=g) * (v_max / 4)
    done = (torch.rand(B, generator=g) < 0.3).float()
    k = torch.randint(0, n_atom, (B, ), generator=g)
    rows_of = lambda m: torch.nonzero(m.repeat_interleave(Aa)).reshape(-1)  # noqa: E731
    for r in rows_of(pick['uniform']).tolist():
        dist[r] = torch.softmax(0.1 * torch.randn(N, n_atom, generator=g), -1)
    for r in rows_of(pick['peaked']).tolist():
        dist[r] = torch.softmax(8.0 * torch.randn(N, n_atom, generator=g), -1) + 1e-6
    for nm in ('converged', 'subnormal', 'int_bins'):
        m = pick[nm]
        done[m] = 1.0
        reward[:, m] = 0.0
        reward[0, m] = support[k[m]]
    for r in rows_of(pick['converged']).tolist():
        kk = int(k[r // Aa])
        eps = float(10.0 ** (-6.0 + 3.0 * torch.rand(1, generator=g)))
        row = torch.softmax(torch.randn(n_atom, generator=g), -1) * eps
        row[kk] = 1.0 - eps
        dist[r, act[r]] = row
    for r in rows_of(pick['subnormal']).tolist():
        kk = int(k[r // Aa])
        row = torch.softmax(3.0 * torch.randn(n_atom, generator=g), -1)
        far = (torch.arange(n_atom) - kk).abs() >= 2  # the neighbours of k may get mass when Tz is not exactly on k
        sel = far & (torch.rand(n_atom, generator=g) < 0.3)
        if far.any():
            sel[torch.nonzero(far).reshape(-1)[0]] = True
        row[sel] = SUBNORMALS[torch.randint(0, 3, (int(sel.sum()), ), generator=g)]
        assert not sel[kk]
        dist[r, act[r]] = row
    m = pick['clamped']
    reward[:, m] = 0.0
    reward[0, m] = torch.where(torch.rand(int(m.sum()), generator=g) < 0.5, -1e3, 1e3)
    m = pick['reversed']
    done[m] = 3.0 * torch.randn(int(m.sum()), generator=g)
    if zeros:
        for r in rows_of(pick['zeros']).tolist():
            row = dist[r, act[r]]
            row[torch.rand(n_atom, generator=g) < 0.2] = 0.0
            row[int(torch.randint(0, n_atom, (1, ), generator=g))] = 0.0
    t = OrderedDict()
    lead = (B, ) if A is None else (B, A)
    t['dist'] = dist.reshape(*lead, N, n_atom)
    nk = 'next_dist' if one_step else 'next_n_dist'
    t[nk] = ndist.reshape(*lead, N, n_atom)
    t['act'] = act.reshape(lead)
    t['next_act' if one_step else 'next_n_act'] = nact.reshape(lead)
    p = dict(gamma=0.99, v_min=v_min, v_max=v_max, n_atom=n_atom)
    meta = dict(regime=reg.repeat_interleave(Aa).numpy(), names=names, R=R, N=N, n_atom=n_atom, nk=nk)
    if one_step:
        t['reward'] = reward[0]
        t['done'] = done
        t['weight'] = None
        return 'd1td', t, p, meta
    t['reward'] = reward
    t['done'] = done
    if weight == 'tensor':
        t['weight'] = _zeros_at(g, torch.rand(R, generator=g), 0.05)
    elif weight == 'one':
        t['weight'] = torch.rand(1, generator=g)
    else:
        t['weight'] = None
        if weight == 'float':
            p['weight_float'] = 0.7
    p['nstep'] = nstep
    if vg == 'tensor':
        t['value_gamma'] = torch.rand(B, generator=g) * 0.2 + 0.8
        t['value_gamma'][pick['reversed'] & (torch.rand(B, generator=g) < 0.5)] *= -1.0
    elif vg == '0dim':
        t['value_gamma'] = torch.tensor(0.9)
    elif vg == 'float':
        p['value_gamma'] = 0.857
    return 'dntd', t, p, meta


# ----------------------------------------------------------------------------------------------------------------
# QR-DQN / IQN / FQF (quantile_td_kernel)
# ----------------------------------------------------------------------------------------------------------------
QT_REGIMES = ('live', 'fractional', 'tie', 'kappa_edge')


def gen_qt(seed, kind, B, N, n, n_p, nstep, kappa=1.0, tau='tensor', vg=None, weight=True):
    """live: done 0; fractional: done in (0, 1); tie: done 1 and a dyadic target r0, half the chosen quantiles equal to r0
    (u == 0 exactly); kappa_edge: done 1, target 0, half the chosen quantiles at +-(the Huber threshold) (|u| == kappa
    exactly: fp32(kappa) for IQN, 1 for the smooth-l1 of QR-DQN / FQF)."""
    g = cases._g(seed)
    reg = _regimes(g, B, QT_REGIMES)
    pick = {nm: reg == i for i, nm in enumerate(QT_REGIMES)}
    theta = torch.randn(B, N, n, generator=g)  # canonical (sample, action, quantile)
    ntheta = torch.randn(B, N, n_p, generator=g)
    act = torch.randint(0, N, (B, ), generator=g)
    nact = torch.randint(0, N, (B, ), generator=g)
    reward = torch.rand(nstep, B, generator=g) * 2.0 - 1.0
    done = torch.zeros(B)
    done[pick['fractional']] = torch.rand(B, generator=g)[pick['fractional']]
    edge = float(np.float32(kappa)) if kind == 'iqn' else 1.0
    r0 = _dyadic(g, B)
    for b in range(B):
        if pick['tie'][b] or pick['kappa_edge'][b]:
            done[b] = 1.0
            reward[:, b] = 0.0
            half = torch.rand(n, generator=g) < 0.5
            half[0] = True
            if pick['tie'][b]:
                reward[0, b] = r0[b]
                theta[b, act[b], half] = r0[b]
            else:
                theta[b, act[b], half] = torch.where(torch.rand(int(half.sum()), generator=g) < 0.5, -edge, edge)
    perm = {'qrdqn': (0, 1, 2), 'iqn': (2, 0, 1), 'fqf': (0, 2, 1)}[kind]
    t = OrderedDict()
    t['q'] = theta.permute(*perm).contiguous()
    t['next_n_q'] = ntheta.permute(*perm).contiguous()
    t['action'] = act
    t['next_n_action'] = nact
    t['reward'] = reward
    t['done'] = done
    if kind == 'qrdqn':
        mid = (torch.arange(n, dtype=torch.float32) + 0.5) / n
        t['tau'] = {'tensor': torch.rand(B, n, 1, generator=g), 'row': mid.view(1, n, 1), 'scalar': torch.tensor(0.3)}[tau]
    elif kind == 'iqn':
        t['replay_quantiles'] = torch.rand(n, B, 1, generator=g)
    else:
        t['quantiles_hats'] = torch.rand(B, n, generator=g).sort(dim=1).values
    t['weight'] = _zeros_at(g, torch.rand(B, generator=g) + 0.5, 0.05) if weight else None
    p = dict(gamma=0.99, nstep=nstep)
    if kind != 'qrdqn':
        p['kappa'] = kappa
    if vg == 'tensor':
        t['value_gamma'] = torch.rand(B, generator=g) * 0.2 + 0.8
    elif vg == '0dim':
        t['value_gamma'] = torch.tensor(0.9)
    return kind, t, p, dict(regime=reg.numpy(), names=QT_REGIMES)


# ----------------------------------------------------------------------------------------------------------------
# TD(lambda) (lambda_scan_kernel, loss head)
# ----------------------------------------------------------------------------------------------------------------
def gen_tdl(seed, T, B):
    g = cases._g(seed)
    t = OrderedDict()
    t['value'] = torch.randn(T + 1, B, generator=g)
    t['reward'] = torch.rand(T, B, generator=g)
    t['weight'] = _zeros_at(g, torch.rand(T, B, generator=g), 0.05)
    reg = (t['weight'] == 0).reshape(-1).long().numpy()
    return 'td_lambda', t, dict(gamma=0.997, lambda_=0.99), dict(regime=reg, names=('weighted', 'zero_weight'))


# ----------------------------------------------------------------------------------------------------------------
# the cases: every geometry hand-off of the kernels
# ----------------------------------------------------------------------------------------------------------------
CASES = OrderedDict([
    # qntd: one CTA up to S = 1024, the one-round-trip grid sum up to 511 CTAs (S = 65408), the ticketed sum above
    ('qntd_mse_n1_S1', lambda: gen_qn(8001, 1, 4, 1)),
    ('qntd_l1_n8_S1024_vgT', lambda: gen_qn(8002, 1024, 6, 8, crit='l1', vg='tensor')),
    ('qntd_smoothl1_n9_S1025_vg0', lambda: gen_qn(8003, 1025, 6, 9, crit='smoothl1', vg='0dim')),
    ('qntd_huber_n12_S65408_vgF', lambda: gen_qn(8004, 65408, 4, 12, crit='huber', vg='float')),
    ('qntd_mse_n12_S65409_nw', lambda: gen_qn(8005, 65409, 4, 12, weight=False)),
    ('qntd_huber_n9_S100003_vgT', lambda: gen_qn(8006, 100003, 3, 9, crit='huber', vg='tensor')),
    ('qntd_l1_n1_S100003', lambda: gen_qn(8007, 100003, 3, 1, crit='l1')),
    ('qntd_rescale_n8_S1025_vgT', lambda: gen_qn(8010, 1025, 6, 8, rescale=True, vg='tensor')),
    ('qntd_rescale_n12_S65409', lambda: gen_qn(8011, 65409, 4, 12, rescale=True)),
    ('qntd_rescale_huber_n9_S1024', lambda: gen_qn(8012, 1024, 5, 9, rescale=True, crit='huber')),
    ('bdq_G3_n9_S1025_vgT', lambda: gen_qn(8020, 1025, 5, 9, vg='tensor', G=3)),
    ('bdq_G4_n12_S65409_smoothl1', lambda: gen_qn(8021, 65409, 3, 12, crit='smoothl1', G=4)),
    ('marl_A3_n9_S4099_vgT', lambda: gen_qn(8030, 4099, 5, 9, vg='tensor', marl=True)),
    ('qseq_T8_B129_n9', lambda: gen_qseq(8040, 8, 129, 6, 9, rescale=False)),
    ('qseq_T5_B205_n12_rescale', lambda: gen_qseq(8041, 5, 205, 4, 12, rescale=True)),
    ('q1td_S1025', lambda: gen_sibling(8050, 'q1td', 1025, N=6)),
    ('v1td_S65409', lambda: gen_sibling(8051, 'v1td', 65409)),
    ('vntd_n12_S4099', lambda: gen_sibling(8052, 'vntd', 4099, nstep=12)),
    # C51: 256 / 128 threads at R = 4088 / 4089, 2 / 8 atoms per lane at n_atom 64 / 65, the cap at 256
    ('dntd_a2_n1_R4088', lambda: gen_dn(8100, 4088, 3, 2, 1, vg='tensor')),
    ('dntd_a32_n3_R4089', lambda: gen_dn(8101, 4089, 3, 32, 3, weight='float')),
    ('dntd_a33_n8_R1031_c51', lambda: gen_dn(8102, 1031, 4, 33, 8, vrange='c51', vg='0dim')),
    ('dntd_a51_n9_R4088_c51', lambda: gen_dn(8103, 4088, 3, 51, 9, vrange='c51', vg='tensor')),
    ('dntd_a51_n12_R8197', lambda: gen_dn(8104, 8197, 2, 51, 12, vg='float', weight='one')),
    ('dntd_a64_n9_R4089', lambda: gen_dn(8105, 4089, 2, 64, 9, vg='tensor')),
    ('dntd_a65_n12_R4088', lambda: gen_dn(8106, 4088, 2, 65, 12, weight='none')),
    ('dntd_a200_n3_R2053_c51', lambda: gen_dn(8107, 2053, 3, 200, 3, vrange='c51', vg='tensor')),
    ('dntd_a256_n12_R4089', lambda: gen_dn(8108, 4089, 2, 256, 12, vg='tensor')),
    ('dntd_marl_A3_a51_n9_R4089', lambda: gen_dn(8109, 1363, 3, 51, 9, A=3, vg='0dim')),
    ('d1td_a51_R4089_zeros', lambda: gen_dn(8110, 4089, 3, 51, 1, vrange='c51', one_step=True, zeros=True)),
    ('d1td_marl_A2_a65_R2050_zeros', lambda: gen_dn(8111, 1025, 3, 65, 1, A=2, one_step=True, zeros=True)),
    # quantile heads: 1 / 32 / 200 / 2048 quantiles on either axis, kappa 0.3 / 1 / 1.7, nstep up to 12
    ('qrdqn_200x200_n3_tauT', lambda: gen_qt(8200, 'qrdqn', 64, 4, 200, 200, 3, tau='tensor')),
    ('qrdqn_1x2048_n9_tauS', lambda: gen_qt(8201, 'qrdqn', 32, 3, 1, 2048, 9, tau='scalar', vg='tensor')),
    ('qrdqn_2048x32_n12_tauR', lambda: gen_qt(8202, 'qrdqn', 16, 3, 2048, 32, 12, tau='row', vg='0dim')),
    ('qrdqn_2048x2048_n1', lambda: gen_qt(8203, 'qrdqn', 4, 2, 2048, 2048, 1)),
    ('iqn_32x32_n9_k0.3', lambda: gen_qt(8210, 'iqn', 257, 5, 32, 32, 9, kappa=0.3, vg='tensor')),
    ('iqn_200x200_n3_k1.7', lambda: gen_qt(8211, 'iqn', 33, 4, 200, 200, 3, kappa=1.7)),
    ('iqn_2048x1_n12_k1', lambda: gen_qt(8212, 'iqn', 16, 3, 2048, 1, 12, kappa=1.0, vg='0dim')),
    ('iqn_2048x2048_n5_k0.3', lambda: gen_qt(8213, 'iqn', 4, 2, 2048, 2048, 5, kappa=0.3)),
    ('fqf_32x200_n12_k1.7', lambda: gen_qt(8220, 'fqf', 65, 4, 32, 200, 12, kappa=1.7, vg='tensor')),
    ('fqf_1x1_n1_k0.3', lambda: gen_qt(8221, 'fqf', 1025, 3, 1, 1, 1, kappa=0.3)),
    ('fqf_200x2048_n8_k1', lambda: gen_qt(8222, 'fqf', 8, 3, 200, 2048, 8, kappa=1.0, weight=False)),
    # TD(lambda): 8-column tiles below B = 4224 (16 * 2 * 132 SMs), 16-column tiles from there
    ('tdl_T1_B4223', lambda: gen_tdl(8300, 1, 4223)),
    ('tdl_T1024_B4224', lambda: gen_tdl(8301, 1024, 4224)),
    ('tdl_T4096_B4223', lambda: gen_tdl(8302, 4096, 4223)),
    ('tdl_T4096_B4224', lambda: gen_tdl(8303, 4096, 4224)),
])


# ----------------------------------------------------------------------------------------------------------------
# per-row views, branch boundaries, regime fractions
# ----------------------------------------------------------------------------------------------------------------
def row_view(op, key, x):
    """``x`` with one row per regime row on axis 0, or None for outputs that are not per row"""
    x = np.asarray(x)
    if key in ('out_loss', 'out_priority') or x.ndim == 0:
        return None
    if op == 'qseq':
        return x.reshape((-1, ) + x.shape[2:])
    if op == 'iqn' and key == 'grad_q':
        return np.moveaxis(x, 1, 0)
    if op in ('dntd', 'd1td') and key == 'grad_dist':
        return x.reshape((-1, ) + x.shape[-2:])
    if op == 'td_lambda':  # value (T+1, B): the last row gets no gradient; regimes are the (T, B) weights
        return x[:-1].reshape(-1)
    return x


def boundary(op, meta, r64):
    """rows whose fp64 gradient sits on a kink that fp32 rounding may put on the other side: an L1 criterion with
    0 < |d| tiny.  (The other criteria, the C51 cross entropy and the quantile Huber terms have continuous gradients.)"""
    if op == 'qntd' and meta.get('crit') == 'l1':
        per = np.asarray(r64['out_td_error_per_sample']).reshape(len(meta['regime']), -1)
        return ((per > 0) & (per < 1e-5)).any(1)
    return None


def regime_fractions(meta):
    reg = meta['regime']
    return {nm: float(np.mean(reg == i)) for i, nm in enumerate(meta['names'])}


@functools.lru_cache(maxsize=2)
def _case(name):
    op, t, p, meta = CASES[name]()
    refs = {path: run_ref(op, t, p, path) for path in PATHS}
    return op, t, p, meta, refs


def _dntd_checks(tag, t, p, meta, got, stash):
    R, N, na = meta['R'], meta['N'], meta['n_atom']
    act = t['act'].reshape(R).numpy()
    gd = np.asarray(got['grad_dist']).reshape(R, N, na)
    off = np.ones((R, N), bool)
    off[np.arange(R), act] = False
    assert np.all(gd[off] == 0.0), (tag, 'gradient off the chosen action')
    if 'proj' not in stash:
        return
    proj = stash['proj']
    nd = t['next_n_dist'].reshape(R, N, na).double().numpy()[np.arange(R), t['next_n_act'].reshape(R).numpy()]
    want = nd.sum(1)
    err = np.abs(proj.sum(1) - want)
    assert np.all(err <= 4 * na * EPS32 * want), (tag, 'projected mass not conserved', float(err.max()))
    assert np.all(proj >= 0), (tag, 'negative projected mass')
    d = t['dist'].reshape(R, N, na).double().numpy()[np.arange(R), act]
    below = (d <= 1.0).all(1)
    td = np.asarray(got['out_td_error_per_sample']).reshape(R)
    assert np.all(td[below] >= 0.0), (tag, 'negative TD error with dist <= 1', float(td[below].min()))


def _compare_case(tag, op, meta, got, r32, r64):
    bnd = boundary(op, meta, r64)
    with np.errstate(invalid='ignore'):  # dist_1step_td_error rows with a zero probability: inf - inf where both are inf
        return _compare_rows(tag, op, meta, got, r32, r64, bnd)


def _compare_rows(tag, op, meta, got, r32, r64, bnd):
    worst = compare64(tag, got, r32, r64, bnd=bnd, S=len(meta['regime']))
    reg = meta['regime']
    keys = [k for k in r64 if row_view(op, k, r64[k]) is not None]
    for i, nm in enumerate(meta['names']):
        m = reg == i
        if not m.any() or m.all():
            continue
        sub = [OrderedDict((k, row_view(op, k, d[k])[m]) for k in keys) for d in (got, r32, r64)]
        worst = max(worst, compare64('%s [%s]' % (tag, nm), *sub, bnd=None if bnd is None else bnd[m]))
    return worst


# ----------------------------------------------------------------------------------------------------------------
# CPU: the generators reach every regime, the reference is float64, the fp32 oracle is a sane yardstick
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', list(CASES))
def test_reference_fp64(name):
    op, t, p, meta, refs = _case(name)
    if len(meta['regime']) >= 100:
        frac = regime_fractions(meta)
        assert min(frac.values()) >= REGIME_MIN, (name, frac)
    for path, (r32, r64) in refs.items():
        assert set(r32) == set(r64)
        for k, v in r64.items():
            assert np.asarray(v).dtype == np.float64, (name, path, k, np.asarray(v).dtype)
        worst = 0.0
        for k in r64:
            a, b = np.asarray(r32[k], np.float64), np.asarray(r64[k], np.float64)
            fin = np.isfinite(b)
            assert np.array_equal(fin, np.isfinite(a)), (name, path, k, 'fp32 oracle non-finite pattern')
            if not fin.any():
                continue
            scale = float(np.abs(b[fin]).max())
            keep = fin & np.isfinite(a)
            e32 = float(np.abs(a[keep] - b[keep]).max()) if keep.any() else 0.0
            assert e32 <= SANE * scale, (name, path, k, e32, scale)
            worst = max(worst, e32 / (EPS32 * scale) if scale > 0 else 0.0)
        print('\n[fp64 ref] %-36s %-5s max |fp32 oracle - fp64| = %.1f * 2^-24 * scale' % (name, path, worst))


def test_regime_checks_are_real():
    """the data of the special regimes really is what the comparison rests on"""
    _, t, _, meta = gen_qn(8003, 1025, 6, 9, crit='smoothl1', vg='0dim')
    th = meta['regime'] == meta['names'].index('threshold')
    qsa = t['q'][torch.arange(1025), t['action']]
    assert torch.equal((qsa - t['reward'][0])[torch.from_numpy(th)].abs(), torch.full((int(th.sum()), ), 2.0))
    _, t, _, meta = gen_qt(8211, 'iqn', 33, 4, 200, 200, 3, kappa=1.7)
    theta = t['q'].permute(1, 2, 0)[torch.arange(33), t['action']]  # (B, n)
    tie = torch.from_numpy(meta['regime'] == meta['names'].index('tie'))
    edge = torch.from_numpy(meta['regime'] == meta['names'].index('kappa_edge'))
    assert ((theta[tie] - t['reward'][0][tie].unsqueeze(1)) == 0).any(1).all()
    assert (theta[edge].abs() == np.float32(1.7)).any(1).all()
    _, t, p, meta = gen_dn(8103, 4088, 3, 51, 9, vrange='c51', vg='tensor')
    sub = torch.from_numpy(meta['regime'] == meta['names'].index('subnormal'))
    d = t['dist'][torch.arange(4088), t['act']][sub]
    tiny = (d > 0) & (d < torch.finfo(torch.float32).tiny)
    assert tiny.any(1).all()
    rev = torch.from_numpy(meta['regime'] == meta['names'].index('reversed'))
    assert ((1 - t['done'][rev]) * t['value_gamma'][rev] < 0).float().mean() > 0.3


# ----------------------------------------------------------------------------------------------------------------
# GPU
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('name', list(CASES))
def test_value_td_fp64(name):
    op, t, p, meta, refs = _case(name)
    for path in PATHS:
        got, stash = run_gpu(op, t, p, path)
        r32, r64 = refs[path]
        tag = '%s %s' % (name, path)
        _compare_case(tag, op, meta, got, r32, r64)
        if op in ('dntd', 'd1td'):
            _dntd_checks(tag, t, p, meta, got, stash)


@pytest.mark.gpu
@pytest.mark.parametrize('kind', ['qrdqn', 'iqn', 'fqf'])
@pytest.mark.parametrize('axis', ['n_tau', 'n_tau_prime'])
def test_quantile_rejects_2049(kind, axis):
    """one CTA keeps every quantile of a sample in shared memory: 2048 is the cap, 2049 is an error (never a silent
    truncation)"""
    import di_engine_b200 as b2
    from di_engine_b200 import _lib
    n, n_p = (2049, 8) if axis == 'n_tau' else (8, 2049)
    op, t, p, _ = gen_qt(8230, kind, 4, 2, n, n_p, 1, kappa=1.0)
    with pytest.raises(_lib.B200RLError):
        cases.run_api(b2.rl_utils, op, t, p, device=DEV)
