"""The continuous-action policy-gradient losses on csrc/heads.cu: ``a2c_error_continuous`` (ding/rl_utils/a2c.py:50-88, the
a2cc_kernel) and ``ppo_policy_error_continuous`` (ding/rl_utils/ppo.py:377-450, the ppoc_kernel with a zero value head).

CPU (``-m "not gpu"``):
  * the fixtures in ``tests/golden/pg_continuous/`` hold the seeded inputs, and the live reference reproduces their outputs;
  * every public call marshals against the ctypes prototypes (recording stand-in of test_reference_suite.py);
  * the reference's assertions and errors hold (dual_clip <= 1, an unknown kl_type, shape mismatches), and ``kl_div`` is the
    python int 0 without a pretrained policy;
  * the reference's own ``test_a2c_continuous`` runs against the reference and the stand-in.
GPU: every output and the gradients of mu, sigma (and value), for unit, mixed and repeated upstream gradients, against the
fixtures (minted from the unmodified reference by ``tests/golden/make_pg_continuous_golden.py``), against the live reference
from ``oracle/_ref`` on CUDA tensors, and against a float64 restatement on off-policy batches, at 1e-5 with gradients scaled
by their largest magnitude; and the policy lines of A2C, PPOPG and PPOOff (continuous, hybrid) before and after ``install()``.
"""
import contextlib
import glob
import json
import math
import os

import numpy as np
import pytest
import torch

import di_engine_b200 as b2
from di_engine_b200 import ops
from oracle import ref_loader
from tests.test_reference_suite import _RecordingLib

HAVE_REF = ref_loader.available()
GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'pg_continuous')
FIELDS = {
    'a2c': ('mu', 'sigma', 'action', 'value', 'adv', 'return_', 'weight'),
    'ppo': ('mu', 'sigma', 'mu_old', 'sigma_old', 'action', 'adv', 'weight', 'mu_pre', 'sigma_pre'),
}
OUTS = {'a2c': ('policy', 'value', 'entropy'), 'ppo': ('policy', 'entropy', 'kl', 'approx_kl', 'clipfrac')}
GRADS = {'a2c': ('mu', 'sigma', 'value'), 'ppo': ('mu', 'sigma')}
# upstream gradient of each loss for the 'mix' runs; none of them is a loss weight the forward launch expects
MIX = {'a2c': (1.3, 0.7, -0.02), 'ppo': (1.3, -0.02, 0.4)}


def _case(fn, seed, B, D, weight=True, clip=0.2, dual=None, kl=None, old1d=False, rows='plain'):
    """rows: 'plain' (sigma = exp(0.5 randn), actions drawn from the policy), 'wide' (sigma from 1e-3 to 1e2, actions 3 to 6
    sigma from mu), 'grid' (D = 1: a quarter of the rows has a ratio of exactly fp32(1 + clip), a quarter exactly
    fp32(1 - clip)), 'far' (off-policy: old policies far from the new one, many ratios clipped)"""
    return dict(fn=fn, seed=seed, B=B, D=D, weight=weight, clip=clip, dual=dual, kl=kl, old1d=old1d, rows=rows)


def _boundary_rows(target, lo_side):
    """(sigma, t) pairs, both fp32, for which the reference's fp32 ratio exp(lp_new - lp_old) is exactly fp32(target): one
    action dim, sigma shared by both policies, the action at one mean and the other mean t away (lp as Normal.log_prob
    computes it).  The log-ratio is an fp32 number, and only two to four of them round to the target under exp; kept are
    the pairs whose log-ratio has an exact exp within 0.2 ulp of the target, and whose sigma has an exact log within 0.1 ulp
    of its fp32 log, so that any expf / logf with a smaller error than that lands on the same ratio"""
    c = torch.tensor(math.log(math.sqrt(2 * math.pi)), dtype=torch.float32)
    goal = torch.tensor(target, dtype=torch.float32)
    sig = torch.linspace(0.05, 4.0, 4000, dtype=torch.float32)
    L = torch.log(sig)
    ok = np.abs(np.log(sig.double().numpy()) - L.double().numpy()) < 0.1 * np.spacing(np.abs(L.numpy()))
    sig, L = sig[torch.from_numpy(ok)].unsqueeze(1), L[torch.from_numpy(ok)].unsqueeze(1)
    x0 = math.sqrt(2 * abs(math.log(target)))
    t = (x0 + torch.arange(-64, 64, dtype=torch.float32) * 2.0 ** -24) * sig
    s = sig.expand_as(t)
    lp_t = -(t * t) / (2 * (s * s)) - L - c
    lp_0 = -(torch.zeros_like(t) ** 2) / (2 * (s * s)) - L - c
    d = (lp_t - lp_0) if lo_side else (lp_0 - lp_t)
    ulp = float(np.spacing(np.float32(target)))
    exact = torch.from_numpy(np.abs(np.exp(d.double().numpy()) - float(goal)) < 0.2 * ulp)
    hit = (torch.exp(d) == goal) & exact
    assert int(hit.sum()) >= 4, (target, int(hit.sum()))
    return s[hit], t[hit]


def make_inputs(c):
    g = torch.Generator().manual_seed(c['seed'])
    B, D = c['B'], c['D']

    def randn(*s):
        return torch.randn(*s, generator=g)

    def rand(*s):
        return torch.rand(*s, generator=g)

    t = {}
    mu = randn(B, D)
    if c['rows'] == 'wide':
        sigma = 10.0 ** (rand(B, D) * 5.0 - 3.0)
        sign = torch.where(rand(B, D) < 0.5, -1.0, 1.0)
        action = mu + sigma * sign * (3.0 + 3.0 * rand(B, D))
    else:
        sigma = torch.exp(0.5 * randn(B, D))
        action = mu + sigma * randn(B, D)
    adv = randn(B)
    adv[rand(B) < 0.2] = 0.0
    t.update(mu=mu, sigma=sigma, action=action, adv=adv)
    if c['fn'] == 'a2c':
        t['value'] = randn(B)
        t['return_'] = 2.0 * randn(B)
    else:
        if c['rows'] == 'far':
            t['mu_old'] = mu + 0.5 * sigma * randn(B, D)
            t['sigma_old'] = sigma * torch.exp(0.3 * randn(B, D))
        elif c['rows'] == 'wide':  # per-dimension log-ratios of order 1 at every scale
            t['mu_old'] = mu + 0.1 * sigma * randn(B, D)
            t['sigma_old'] = sigma * torch.exp(0.05 * randn(B, D))
        else:  # near-on-policy: the log-ratio summed over D dims stays of order 0.1 at every D
            k = 0.1 / max(1.0, D / 6) ** 0.5
            t['mu_old'] = mu + k * sigma * randn(B, D)
            t['sigma_old'] = sigma * torch.exp(k * randn(B, D))
        if c['rows'] == 'grid':
            assert D == 1
            q = B // 4
            zero = torch.zeros(q, 1)
            # ratio 1 + clip: new mean at the action, old mean t away; 1 - clip: the other way round
            s_hi, t_hi = _boundary_rows(1.0 + c['clip'], False)
            k = torch.randint(0, s_hi.numel(), (q, ), generator=g)
            t['mu'][:q], t['sigma'][:q], t['action'][:q] = zero, s_hi[k].reshape(-1, 1), zero
            t['mu_old'][:q], t['sigma_old'][:q] = t_hi[k].reshape(-1, 1), s_hi[k].reshape(-1, 1)
            s_lo, t_lo = _boundary_rows(1.0 - c['clip'], True)
            k = torch.randint(0, s_lo.numel(), (q, ), generator=g)
            t['mu'][q:2 * q], t['sigma'][q:2 * q], t['action'][q:2 * q] = t_lo[k].reshape(-1, 1), s_lo[k].reshape(-1, 1), zero
            t['mu_old'][q:2 * q], t['sigma_old'][q:2 * q] = zero, s_lo[k].reshape(-1, 1)
        if c['old1d']:
            t['mu_old'], t['sigma_old'] = t['mu_old'].reshape(B), t['sigma_old'].reshape(B)
        if c['kl']:
            t['mu_pre'] = mu + 0.3 * sigma * randn(B, D)
            t['sigma_pre'] = sigma * torch.exp(0.1 * randn(B, D))
        else:
            t['mu_pre'] = t['sigma_pre'] = None
    t['weight'] = rand(B) + 0.5 if c['weight'] else None
    return t


# fixture cases (tests/golden/pg_continuous/<name>.npz); the shipped shapes: A2C on Pendulum B = 32, D = 1 and on BipedalWalker
# B = 256, D = 4; PPOPG on BipedalWalker B = 64, D = 4; the hybrid action's continuous part B = 320, D = 2
CASES = {
    'a2c_pendulum': _case('a2c', 1, 32, 1, weight=False),
    'a2c_bipedal': _case('a2c', 2, 256, 4),
    'a2c_b1': _case('a2c', 3, 1, 3),
    'a2c_d17': _case('a2c', 4, 129, 17, weight=False),
    'a2c_d32': _case('a2c', 5, 64, 32),
    'a2c_wide': _case('a2c', 6, 257, 6, rows='wide'),
    'ppo_bipedal': _case('ppo', 11, 64, 4, weight=False),
    'ppo_hybrid': _case('ppo', 12, 320, 2),
    'ppo_b1': _case('ppo', 13, 1, 3),
    'ppo_d32_dual': _case('ppo', 14, 64, 32, dual=3.0),
    'ppo_clip01': _case('ppo', 15, 129, 6, clip=0.1, weight=False),
    'ppo_far_dual': _case('ppo', 16, 513, 3, dual=3.0, rows='far'),
    'ppo_far_clip01': _case('ppo', 17, 513, 6, clip=0.1, rows='far'),
    'ppo_wide': _case('ppo', 18, 257, 3, rows='wide'),
    'ppo_old1d': _case('ppo', 19, 64, 1, old1d=True),
    'ppo_old1d_noweight': _case('ppo', 20, 33, 1, old1d=True, weight=False, dual=3.0),
    'ppo_pre_k1': _case('ppo', 21, 64, 4, kl='k1'),
    'ppo_pre_k2': _case('ppo', 22, 64, 17, kl='k2', dual=3.0),
    'ppo_pre_k3': _case('ppo', 23, 129, 6, kl='k3', rows='far'),
    'ppo_grid': _case('ppo', 24, 256, 1, rows='grid'),
    'ppo_grid_clip01_dual': _case('ppo', 25, 256, 1, clip=0.1, dual=3.0, rows='grid'),
}


def run(api, c, t, dev, grad='mix'):
    """call the public function of ``api`` (the reference or ours) on case ``c``; grad: 'unit' (the sum of the losses), 'mix'
    (MIX) or 'repeat' (MIX, backward twice through the same graph) -> dict of numpy outputs + gradients"""
    d = {k: (v.to(dev) if isinstance(v, torch.Tensor) else v) for k, v in t.items()}
    leaves = {k: d[k].clone().requires_grad_(True) for k in GRADS[c['fn']]}
    new = {'mu': leaves['mu'], 'sigma': leaves['sigma']}
    if c['fn'] == 'a2c':
        losses = list(api.a2c_error_continuous(api.a2c_data(new, d['action'], leaves['value'], d['adv'], d['return_'],
                                                            d['weight'])))
        res = dict(zip(OUTS['a2c'], losses))
    else:
        pre = {'mu': d['mu_pre'], 'sigma': d['sigma_pre']} if c['kl'] else None
        data = api.ppo_policy_data_continuous(new, {'mu': d['mu_old'], 'sigma': d['sigma_old']}, d['action'], d['adv'],
                                              d['weight'], pre)
        kw = dict(clip_ratio=c['clip'], dual_clip=c['dual'])
        if c['kl']:
            kw['kl_type'] = c['kl']
        loss, info = api.ppo_policy_error_continuous(data, **kw)
        losses = list(loss)
        if not c['kl']:
            assert type(loss.kl_div) is int and loss.kl_div == 0
            losses = losses[:2]
        res = dict(policy=loss.policy_loss, entropy=loss.entropy_loss, kl=loss.kl_div.detach() if c['kl'] else torch.tensor(0.0),
                   approx_kl=torch.tensor(info.approx_kl), clipfrac=torch.tensor(info.clipfrac))
        assert isinstance(info.approx_kl, float) and isinstance(info.clipfrac, float)
    assert all(x.shape == () for x in losses)
    if grad == 'unit':
        sum(losses).backward()
    else:
        total = sum(m * x for m, x in zip(MIX[c['fn']], losses))
        total.backward(retain_graph=grad == 'repeat')
        if grad == 'repeat':
            total.backward()
    out = {k: v.detach().cpu().numpy().astype(np.float64) for k, v in res.items()}
    for k, v in leaves.items():
        out['grad_' + k] = v.grad.detach().cpu().numpy().astype(np.float64)
    return out


def compare(got, want, tol=1e-5):
    assert set(got) >= set(want), set(want) - set(got)
    for k in want:
        a, b = np.asarray(got[k], np.float64), np.asarray(want[k], np.float64)
        assert a.shape == b.shape, (k, a.shape, b.shape)
        fin = b[np.isfinite(b)]
        scale = max(1.0, float(np.max(np.abs(fin)))) if k.startswith('grad') and fin.size else 1.0
        assert np.allclose(a, b, rtol=tol, atol=tol * scale, equal_nan=True), (k, float(np.nanmax(np.abs(a - b))))


def load_fixture(name):
    with np.load(os.path.join(GOLDEN_DIR, name + '.npz'), allow_pickle=False) as z:
        d = {k: z[k] for k in z.files}
    case = json.loads(str(d.pop('case')))
    t = {k: (torch.from_numpy(d['in_' + k]) if 'in_' + k in d else None) for k in FIELDS[case['fn']]}
    want = {k: d['out_' + k] for k in OUTS[case['fn']] + tuple('grad_' + g for g in GRADS[case['fn']])}
    return case, t, want


def fixture_names():
    return sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN_DIR, '*.npz'))
                  if not os.path.basename(p).startswith('ported_'))


# =================================================================================================================
# CPU
# =================================================================================================================
def test_fixture_set_matches_cases():
    assert fixture_names() == sorted(CASES)


@pytest.mark.parametrize('name', sorted(CASES))
def test_fixture_inputs_are_the_seeded_case(name):
    case, t, _ = load_fixture(name)
    assert case == json.loads(json.dumps(CASES[name]))
    want = make_inputs(case)
    for k in FIELDS[case['fn']]:
        if want[k] is None:
            assert t[k] is None, k
        else:
            assert t[k].dtype == want[k].dtype and np.array_equal(t[k].numpy(), want[k].numpy()), k


@pytest.mark.skipif(not HAVE_REF, reason='reference not importable here')
@pytest.mark.parametrize('name', sorted(CASES))
def test_fixture_outputs_are_the_live_reference(name):
    case, t, want = load_fixture(name)
    got = run(ref_loader.load(), case, t, 'cpu')
    for k in want:
        assert np.array_equal(got[k], want[k], equal_nan=True), (name, k)


def test_fixtures_cover_the_edges():
    """the boundary cases hold what their names say, in the stored inputs and reference outputs"""
    for name in ('ppo_grid', 'ppo_grid_clip01_dual'):
        case, t, want = load_fixture(name)
        c = torch.tensor(math.log(math.sqrt(2 * math.pi)), dtype=torch.float32)

        def lp(m, s):
            return (-((t['action'] - m) ** 2) / (2 * s ** 2) - s.log() - c).sum(-1)
        ratio = torch.exp(lp(t['mu'], t['sigma']) - lp(t['mu_old'], t['sigma_old']))
        q = case['B'] // 4
        assert torch.all(ratio[:q] == torch.tensor(1 + case['clip'], dtype=torch.float32))
        assert torch.all(ratio[q:2 * q] == torch.tensor(1 - case['clip'], dtype=torch.float32))
        assert (t['adv'][:2 * q] > 0).any() and (t['adv'][:2 * q] < 0).any() and (t['adv'] == 0).any()
    _, t, _ = load_fixture('a2c_wide')
    assert float(t['sigma'].min()) < 2e-3 and float(t['sigma'].max()) > 50
    z = ((t['action'] - t['mu']) / t['sigma']).abs()
    assert float(z.min()) >= 2.99 and float(z.max()) > 5.9
    _, _, want = load_fixture('ppo_far_dual')
    assert float(want['clipfrac']) > 0.3


@pytest.fixture
def dry(monkeypatch):
    rec = _RecordingLib()
    calls = []

    class _Counting:
        def __getattr__(self, name):
            fn = getattr(rec, name)

            def wrapped(*a):
                calls.append(name)
                return fn(*a)
            return wrapped

    monkeypatch.setattr(ops, 'lib', lambda: _Counting())
    monkeypatch.setattr(ops, 'require_cuda', lambda: None)
    monkeypatch.setattr(ops, 'compute_device', lambda *t: torch.device('cpu'))
    monkeypatch.setattr(ops, 'stream_ptr', lambda: 0)
    monkeypatch.setattr(ops, 'workspace', lambda dev: torch.zeros(1 << 18))
    monkeypatch.setattr(torch.cuda, 'device', lambda d: contextlib.nullcontext())
    monkeypatch.setattr(b2.rl_utils.ppo, 'LAZY_INFO', False)
    yield calls
    ops._CONST.clear()


@pytest.mark.filterwarnings('ignore:invalid value encountered in cast')  # the stand-in leaves outputs uninitialised
@pytest.mark.parametrize('grad', ['mix', 'repeat'])
@pytest.mark.parametrize('name', sorted(CASES))
def test_marshalling_dry_run(dry, name, grad):
    case = CASES[name]
    res = run(b2.rl_utils, case, make_inputs(case), 'cpu', grad)
    entry = 'b200rl_a2c_continuous_fwd_grad' if case['fn'] == 'a2c' else 'b200rl_ppo_continuous_fwd_grad'
    assert dry == [entry] * (3 if grad == 'repeat' else 2), dry
    for k in OUTS[case['fn']]:
        assert res[k].shape == (), k
    B, D = case['B'], case['D']
    assert res['grad_mu'].shape == (B, D) and res['grad_sigma'].shape == (B, D)
    if case['fn'] == 'a2c':
        assert res['grad_value'].shape == (B, )


def test_policy_half_keeps_its_own_gradient_record(dry):
    """ppo_policy_error_continuous and ppo_error_continuous name different expected-upstream-gradient records, so a learner
    that alternates them (PPOOffPolicy) never makes one overwrite the other's; the policy half starts with no value term"""
    seen = []
    orig = ops.head_hint

    def spy(device, kind, init):
        seen.append((kind, list(init)))
        return orig(device, kind, init)
    ops.head_hint = spy
    try:
        t = make_inputs(CASES['ppo_bipedal'])
        new = {'mu': t['mu'], 'sigma': t['sigma']}
        old = {'mu': t['mu_old'], 'sigma': t['sigma_old']}
        b2.ppo_policy_error_continuous(b2.ppo_policy_data_continuous(new, old, t['action'], t['adv'], None, None))
        z = torch.zeros_like(t['adv'])
        b2.ppo_error_continuous(b2.ppo_data(new, old, t['action'], z, z, t['adv'], z, None, None))
        ta = make_inputs(CASES['a2c_bipedal'])
        b2.a2c_error_continuous(b2.a2c_data({'mu': ta['mu'], 'sigma': ta['sigma']}, ta['action'], ta['value'], ta['adv'],
                                            ta['return_'], None))
    finally:
        ops.head_hint = orig
    assert seen == [('ppoc_policy', [1.0, 0.0, -0.01, 0.0]), ('ppoc', [1.0, 0.5, -0.01, 0.0]),
                    ('a2cc', [1.0, 0.5, -0.01, 0.0])], seen


def _apis():
    return [b2.rl_utils] + ([ref_loader.load()] if HAVE_REF else [])


@pytest.mark.filterwarnings('ignore:Using a target size')
def test_error_behaviour_matches_reference(dry):
    """the reference's assertions and errors; where a shape mismatch surfaces in the reference as torch's RuntimeError
    (a broadcast inside the loss), this library raises ValueError before any pointer reaches a kernel, as its other
    operators do"""
    c = CASES['ppo_pre_k1']
    t = make_inputs(c)
    new = {'mu': t['mu'], 'sigma': t['sigma']}
    old = {'mu': t['mu_old'], 'sigma': t['sigma_old']}
    pre = {'mu': t['mu_pre'], 'sigma': t['sigma_pre']}
    B, D = c['B'], c['D']
    for api in _apis():
        data = api.ppo_policy_data_continuous(new, old, t['action'], t['adv'], t['weight'], pre)
        for dc in (1.0, 0.5):  # ppo.py:411-413
            with pytest.raises(AssertionError, match='dual_clip'):
                api.ppo_policy_error_continuous(data, dual_clip=dc)
        with pytest.raises(ValueError, match='kl_type'):  # calculate_kl_div, ppo.py:30-55
            api.ppo_policy_error_continuous(data, kl_type='k4')
        # without a pretrained policy the kl_type is never looked at (ppo.py:443-448)
        loss, _ = api.ppo_policy_error_continuous(data._replace(logit_pretrained=None), kl_type='k4')
        assert type(loss.kl_div) is int and loss.kl_div == 0
        # Normal.log_prob's sample validation in the reference
        with pytest.raises(ValueError):  # a (B, D) policy against a (B, D + 1) action
            api.ppo_policy_error_continuous(data._replace(action=torch.zeros(B, D + 1)))
        with pytest.raises(ValueError):  # old policy of another batch size
            api.ppo_policy_error_continuous(data._replace(mu_sigma_old={'mu': t['mu_old'][:-1],
                                                                        'sigma': t['sigma_old'][:-1]}))
        with pytest.raises(RuntimeError if api is not b2.rl_utils else ValueError):  # adv of another batch size
            api.ppo_policy_error_continuous(data._replace(adv=t['adv'][:-1]))
    c = CASES['a2c_bipedal']
    t = make_inputs(c)
    B, D = c['B'], c['D']
    for api in _apis():
        logit = {'mu': t['mu'], 'sigma': t['sigma']}
        data = api.a2c_data(logit, t['action'], t['value'], t['adv'], t['return_'], t['weight'])
        with pytest.raises(ValueError):
            api.a2c_error_continuous(data._replace(action=torch.zeros(B, D + 1)))
        for k in ('adv', 'value', 'return_', 'weight'):
            with pytest.raises(RuntimeError if api is not b2.rl_utils else ValueError):
                api.a2c_error_continuous(data._replace(**{k: t[k][:-1]}))


def test_namedtuples_and_signatures_match_reference():
    r = b2.rl_utils
    assert r.ppo_data_continuous._fields == ('mu_sigma_new', 'mu_sigma_old', 'action', 'value_new', 'value_old', 'adv',
                                             'return_', 'weight', 'logit_pretrained')  # ppo.py:12-17
    assert r.ppo_policy_data_continuous._fields == ('mu_sigma_new', 'mu_sigma_old', 'action', 'adv', 'weight',
                                                    'logit_pretrained')  # ppo.py:21-23
    import inspect
    sig = [(k, v.default) for k, v in inspect.signature(r.ppo_policy_error_continuous).parameters.items()]
    assert sig == [('data', inspect.Parameter.empty), ('clip_ratio', 0.2), ('dual_clip', None), ('kl_type', 'k1')]
    assert list(inspect.signature(r.a2c_error_continuous).parameters) == ['data']


# ---- the reference's own test, ding/rl_utils/tests/test_a2c.py:31-54, seeded -----------------------------------------------
PORT_FILE = os.path.join(GOLDEN_DIR, 'ported_reference_tests.npz')


def ported_body(api, dev):
    rec = {}
    g = torch.Generator().manual_seed(31)
    random_weight = torch.rand(4, generator=g) + 1
    for i, weight in enumerate([None, random_weight]):
        B, N = 4, 32
        logit = {
            "mu": torch.randn(B, N, generator=g).to(dev).requires_grad_(True),
            "sigma": torch.exp(torch.randn(B, N, generator=g)).to(dev).requires_grad_(True),
        }
        action = torch.randn(B, N, generator=g).to(dev).requires_grad_(True)
        value = torch.randn(B, generator=g).to(dev).requires_grad_(True)
        adv = torch.rand(B, generator=g).to(dev)
        return_ = (torch.randn(B, generator=g) * 2).to(dev)
        data = api.a2c_data(logit, action, value, adv, return_, None if weight is None else weight.to(dev))
        loss = api.a2c_error_continuous(data)
        assert all([l.shape == tuple() for l in loss])
        assert logit["mu"].grad is None
        assert logit["sigma"].grad is None
        assert value.grad is None
        total_loss = sum(loss)
        total_loss.backward()
        assert isinstance(logit["mu"].grad, torch.Tensor)
        assert isinstance(logit['sigma'].grad, torch.Tensor)
        assert isinstance(value.grad, torch.Tensor)
        for k, v in (('policy', loss.policy_loss), ('value', loss.value_loss), ('entropy', loss.entropy_loss),
                     ('grad_mu', logit['mu'].grad), ('grad_sigma', logit['sigma'].grad), ('grad_value', value.grad)):
            rec['%s_%d' % (k, i)] = v.detach().cpu().numpy().astype(np.float64)
    return rec


def _stored_port():
    with np.load(PORT_FILE) as z:
        return {k: z[k] for k in z.files}


@pytest.mark.filterwarnings('ignore:invalid value encountered in cast')
@pytest.mark.parametrize('impl', [
    pytest.param('reference', marks=pytest.mark.skipif(not HAVE_REF, reason='reference not importable here')),
    pytest.param('b200_dry'),
    pytest.param('b200', marks=pytest.mark.gpu),
])
def test_ported_reference_tests(impl, request):
    if impl == 'reference':
        got = ported_body(ref_loader.load(), 'cpu')
        want = _stored_port()
        assert set(got) == set(want)
        for k in want:
            assert np.array_equal(got[k], want[k]), k
    elif impl == 'b200_dry':
        request.getfixturevalue('dry')
        ported_body(b2.rl_utils, 'cpu')
    else:
        got = ported_body(b2.rl_utils, 'cuda')
        compare(got, ported_body(ref_loader.load(), 'cuda') if HAVE_REF else _stored_port())


# =================================================================================================================
# GPU
# =================================================================================================================
def reference_or_skip():
    if not HAVE_REF:
        pytest.skip('reference not importable here')
    return ref_loader.load()


@pytest.mark.gpu
@pytest.mark.parametrize('name', sorted(CASES))
def test_fixture_cases(name):
    case, t, want = load_fixture(name)
    compare(run(b2.rl_utils, case, t, 'cuda'), want)
    if HAVE_REF:
        ref = ref_loader.load()
        for grad in ('unit', 'mix', 'repeat'):
            compare(run(b2.rl_utils, case, t, 'cuda', grad), run(ref, case, t, 'cuda', grad))


SHAPES = [(1, 1), (3, 32), (64, 6), (257, 17), (1025, 3), (4099, 32), (100003, 1), (100003, 6)]


@pytest.mark.gpu
@pytest.mark.parametrize('B,D', SHAPES)
@pytest.mark.parametrize('fn', ['a2c', 'ppo'])
def test_shapes_vs_reference(fn, B, D):
    ref = reference_or_skip()
    seed = 40 + B % 97 + D
    if fn == 'a2c':
        case = _case('a2c', seed, B, D, weight=B % 2 == 0, rows=('plain', 'wide')[seed % 2])
    else:
        case = _case('ppo', seed, B, D, weight=B % 2 == 1, clip=(0.2, 0.1)[seed % 2], dual=(None, 3.0)[D % 2],
                     kl=(None, 'k1', 'k2', 'k3')[seed % 4], rows='far' if D % 2 and D <= 6 else 'plain')
    t = make_inputs(case)
    for grad in ('unit', 'mix'):
        compare(run(b2.rl_utils, case, t, 'cuda', grad), run(ref, case, t, 'cuda', grad))


@pytest.mark.gpu
@pytest.mark.parametrize('name', ['a2c_bipedal', 'ppo_hybrid', 'ppo_pre_k2', 'ppo_old1d'])
def test_host_buffers(name):
    """CPU tensors in: staged to the device, results back on the host, gradients back in the host leaves"""
    case, t, want = load_fixture(name)
    compare(run(b2.rl_utils, case, t, 'cpu'), want)


# ---- float64 restatement on off-policy batches --------------------------------------------------------------------------
def fp64_run(c, t, grad):
    """the two losses restated in float64 from their definitions (Independent(Normal) log-density and entropy, the clipped /
    dual-clipped surrogate, the three KL estimators) with autograd for the gradients"""
    d = {k: (v.double() if isinstance(v, torch.Tensor) else v) for k, v in t.items()}
    leaves = {k: d[k].clone().requires_grad_(True) for k in GRADS[c['fn']]}
    mu, sg = leaves['mu'], leaves['sigma']
    w = d['weight'] if d['weight'] is not None else torch.ones_like(d['adv'])
    half_log_2pi = 0.5 * math.log(2 * math.pi)

    def logp(m, s):
        return (-(d['action'] - m) ** 2 / (2 * s * s) - torch.log(s) - half_log_2pi).sum(-1)
    lp = logp(mu, sg)
    ent = (0.5 + half_log_2pi + torch.log(sg)).sum(-1)
    if c['fn'] == 'a2c':
        v = leaves['value']
        losses = [-(lp * d['adv'] * w).mean(), (w * (d['return_'] - v) ** 2).mean(), (ent * w).mean()]
        res = dict(zip(OUTS['a2c'], losses))
    else:
        mo, so = d['mu_old'].reshape(mu.shape), d['sigma_old'].reshape(mu.shape)
        lpo = logp(mo, so)
        ratio = torch.exp(lp - lpo)
        adv, clip = d['adv'], c['clip']
        sel = torch.min(ratio * adv, ratio.clamp(1 - clip, 1 + clip) * adv)
        if c['dual']:
            sel = torch.max(sel, c['dual'] * adv)
        losses = [-(sel * w).mean(), (ent * w).mean()]
        kl = torch.zeros((), dtype=torch.float64)
        if c['kl']:
            r = lp - logp(d['mu_pre'], d['sigma_pre'])
            kl = {'k1': r.mean(), 'k2': (r ** 2 / 2).mean(), 'k3': (torch.exp(-r) - 1 + r).mean()}[c['kl']]
            losses.append(kl)
        r32 = ratio.detach().float()
        res = dict(policy=losses[0], entropy=losses[1], kl=kl, approx_kl=(lpo - lp).mean(),
                   clipfrac=((r32 > 1 + clip) | (r32 < 1 - clip)).double().mean())
    total = sum(m * x for m, x in zip(MIX[c['fn']], losses)) if grad == 'mix' else sum(losses)
    total.backward()
    out = {k: v.detach().numpy() for k, v in res.items()}
    for k, v in leaves.items():
        out['grad_' + k] = v.grad.numpy()
    return out


FP64_CASES = [
    _case('a2c', 61, 4099, 6, rows='wide'),
    _case('a2c', 62, 100003, 3, weight=False),
    _case('ppo', 63, 4099, 3, dual=3.0, rows='far'),
    _case('ppo', 64, 4099, 6, clip=0.1, rows='far', weight=False),
    _case('ppo', 65, 4099, 3, kl='k3', rows='far'),
    _case('ppo', 66, 100003, 1, kl='k2', dual=3.0, rows='far', old1d=True),
]


@pytest.mark.gpu
@pytest.mark.parametrize('grad', ['unit', 'mix'])
@pytest.mark.parametrize('case', FP64_CASES, ids=lambda c: '%s_B%d_D%d_s%d' % (c['fn'], c['B'], c['D'], c['seed']))
def test_offpolicy_vs_float64(case, grad):
    t = make_inputs(case)
    want = fp64_run(case, t, grad)
    if case['fn'] == 'ppo':
        assert float(want['clipfrac']) > 0.25  # most ratios far from 1: both clip branches and the dual floor run
    got = run(b2.rl_utils, case, t, 'cuda', grad)
    if case['fn'] == 'ppo':  # clipfrac counts the fp32 ratios: a row within an ulp of the boundary may fall either way
        assert abs(float(got.pop('clipfrac')) - float(want.pop('clipfrac'))) * case['B'] <= 2
    compare(got, want)


@pytest.mark.gpu
def test_outputs_are_device_tensors_and_action_gets_no_gradient():
    case, t, _ = load_fixture('a2c_bipedal')
    d = {k: (v.cuda() if v is not None else None) for k, v in t.items()}
    mu, sg, v = (d[k].clone().requires_grad_(True) for k in ('mu', 'sigma', 'value'))
    act = d['action'].clone().requires_grad_(True)
    loss = b2.a2c_error_continuous(b2.a2c_data({'mu': mu, 'sigma': sg}, act, v, d['adv'], d['return_'], d['weight']))
    assert all(x.is_cuda and x.requires_grad for x in loss)
    sum(loss).backward()
    assert act.grad is None  # taken detached (DESIGN section 4)
    assert mu.grad.shape == mu.shape and sg.grad.shape == sg.shape and v.grad.shape == v.shape


# ---- the policy lines, with the reference functions and after install() ------------------------------------------------
def a2c_lines(rl, output, batch, adv_norm, wv, we):
    """ding/policy/a2c.py:164-177 (continuous action space)"""
    adv = batch['adv']
    return_ = batch['value'] + adv
    if adv_norm:
        # norm adv in total train_batch
        adv = (adv - adv.mean()) / (adv.std() + 1e-8)
    error_data = rl.a2c_data(output['logit'], batch['action'], output['value'], adv, return_, batch['weight'])
    a2c_loss = rl.a2c_error_continuous(error_data)
    total_loss = a2c_loss.policy_loss + wv * a2c_loss.value_loss - we * a2c_loss.entropy_loss
    total_loss.backward()
    return total_loss, a2c_loss


def ppopg_lines(rl, output, batch, clip_ratio, entropy_weight):
    """ding/policy/ppo.py:793-804 (continuous action space)"""
    ppo_batch = rl.ppo_policy_data(output['logit'], batch['logit'], batch['action'], batch['return'], batch['weight'], None)
    ppo_loss, ppo_info = rl.ppo_policy_error_continuous(ppo_batch, clip_ratio)
    total_loss = ppo_loss.policy_loss - entropy_weight * ppo_loss.entropy_loss
    total_loss.backward()
    return total_loss, ppo_loss, ppo_info


def ppooff_lines(rl, output, data, adv_norm, clip_ratio, action_space):
    """ding/policy/ppo.py:1276-1311, continuous and hybrid.  The hybrid branch's sum ``type(ppo_continuous_loss)(a, b)``
    builds a three-field ``ppo_policy_loss`` from two values and raises TypeError in the reference; it is run as written and
    must raise the same after install(), and the policy loss is then taken from the two calls' losses."""
    adv = data['adv']
    if adv_norm:
        # Normalize advantage in a total train_batch
        adv = (adv - adv.mean()) / (adv.std() + 1e-8)
    if action_space == 'continuous':
        ppodata = rl.ppo_policy_data(output['logit'], data['logit'], data['action'], adv, data['weight'], None)
        ppo_policy_loss, ppo_info = rl.ppo_policy_error_continuous(ppodata, clip_ratio)
        parts = (ppo_policy_loss, )
    elif action_space == 'hybrid':
        # discrete part (discrete policy loss and entropy loss)
        ppo_discrete_data = rl.ppo_policy_data(
            output['logit']['action_type'], data['logit']['action_type'], data['action']['action_type'], adv,
            data['weight'], None
        )
        ppo_discrete_loss, ppo_discrete_info = rl.ppo_policy_error(ppo_discrete_data, clip_ratio)
        # continuous part (continuous policy loss and entropy loss, value loss)
        ppo_continuous_data = rl.ppo_policy_data(
            output['logit']['action_args'], data['logit']['action_args'], data['action']['action_args'], adv,
            data['weight'], None
        )
        ppo_continuous_loss, ppo_continuous_info = rl.ppo_policy_error_continuous(
            ppo_continuous_data, clip_ratio
        )
        # sum discrete and continuous loss
        with pytest.raises(TypeError):
            ppo_policy_loss = type(ppo_continuous_loss)(
                ppo_continuous_loss.policy_loss + ppo_discrete_loss.policy_loss,
                ppo_continuous_loss.entropy_loss + ppo_discrete_loss.entropy_loss
            )
        ppo_info = type(ppo_continuous_info)(
            max(ppo_continuous_info.approx_kl, ppo_discrete_info.approx_kl),
            max(ppo_continuous_info.clipfrac, ppo_discrete_info.clipfrac)
        )
        parts = (ppo_continuous_loss, ppo_discrete_loss)
    total_loss = sum(p.policy_loss for p in parts) - 0.01 * sum(p.entropy_loss for p in parts)
    total_loss.backward()
    return total_loss, parts, ppo_info


def _policy_runs(rl, seed):
    g = torch.Generator().manual_seed(seed)
    dev = 'cuda'
    out = {}

    def randn(*s):
        return torch.randn(*s, generator=g).to(dev)

    def leaf(x):
        return x.clone().requires_grad_(True)

    for tag, B, D in (('a2c_pendulum', 32, 1), ('a2c_bipedal', 256, 4)):
        mu, sg, v = leaf(randn(B, D)), leaf(torch.exp(0.3 * randn(B, D))), leaf(randn(B))
        batch = {'adv': randn(B), 'value': randn(B), 'action': mu.detach() + sg.detach() * randn(B, D), 'weight': None}
        total, loss = a2c_lines(rl, {'logit': {'mu': mu, 'sigma': sg}, 'value': v}, batch, True, 0.5, 0.01)
        out.update({tag + '_total': total.item(), tag + '_losses': np.array([x.item() for x in loss]),
                    tag + '_grad_mu': mu.grad.cpu().numpy(), tag + '_grad_sigma': sg.grad.cpu().numpy(),
                    tag + '_grad_value': v.grad.cpu().numpy()})
    B, D = 64, 4  # PPOPG on BipedalWalker
    mu, sg = leaf(randn(B, D)), leaf(torch.exp(0.3 * randn(B, D)))
    old = {'mu': mu.detach() + 0.3 * randn(B, D), 'sigma': sg.detach() * torch.exp(0.2 * randn(B, D))}
    batch = {'logit': old, 'action': mu.detach() + sg.detach() * randn(B, D), 'return': randn(B), 'weight': None}
    total, loss, info = ppopg_lines(rl, {'logit': {'mu': mu, 'sigma': sg}}, batch, 0.2, 0.01)
    out.update(ppopg_total=total.item(), ppopg_losses=np.array([loss.policy_loss.item(), loss.entropy_loss.item()]),
               ppopg_info=np.array(list(info)), ppopg_grad_mu=mu.grad.cpu().numpy(), ppopg_grad_sigma=sg.grad.cpu().numpy())
    assert type(loss.kl_div) is int
    for space, B, D in (('continuous', 128, 3), ('hybrid', 320, 2)):
        mu, sg = leaf(randn(B, D)), leaf(torch.exp(0.3 * randn(B, D)))
        old = {'mu': mu.detach() + 0.3 * randn(B, D), 'sigma': sg.detach() * torch.exp(0.2 * randn(B, D))}
        act = mu.detach() + sg.detach() * randn(B, D)
        data = {'adv': randn(B), 'weight': torch.rand(B, generator=g).to(dev) + 0.5}
        if space == 'continuous':
            output = {'logit': {'mu': mu, 'sigma': sg}}
            data.update(logit=old, action=act)
        else:
            lg = leaf(randn(B, 3))
            output = {'logit': {'action_type': lg, 'action_args': {'mu': mu, 'sigma': sg}}}
            data.update(logit={'action_type': lg.detach() + 0.3 * randn(B, 3), 'action_args': old},
                        action={'action_type': torch.randint(0, 3, (B, ), generator=g).to(dev), 'action_args': act})
        total, parts, info = ppooff_lines(rl, output, data, True, 0.2, space)
        out.update({'off_%s_total' % space: total.item(), 'off_%s_info' % space: np.array(list(info)),
                    'off_%s_losses' % space: np.array([x.item() for p in parts for x in (p.policy_loss, p.entropy_loss)]),
                    'off_%s_grad_mu' % space: mu.grad.cpu().numpy(), 'off_%s_grad_sigma' % space: sg.grad.cpu().numpy()})
        if space == 'hybrid':
            out['off_hybrid_grad_logit'] = lg.grad.cpu().numpy()
    return out


@pytest.mark.gpu
def test_policy_lines_before_and_after_install():
    ref = reference_or_skip()
    want = _policy_runs(ref, 77)
    fns = ('a2c_error_continuous', 'ppo_policy_error_continuous', 'ppo_policy_error')
    try:
        b2.install()
        assert all(getattr(ref, n) is getattr(b2.rl_utils, n) for n in fns)
        got = _policy_runs(ref, 77)
        got2 = _policy_runs(ref, 77)  # the second round runs on the upstream gradients the first one recorded
    finally:
        b2.uninstall()
    assert not any(getattr(ref, n) is getattr(b2.rl_utils, n) for n in fns)
    compare(got, want)
    compare(got2, want)
