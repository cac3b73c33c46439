"""The TD losses of the entropy-regularised value learners on the soft_td kernel of csrc/td.cu:
``m_q_1step_td_error`` (Munchausen DQN, ding/rl_utils/td.py:75-158), ``q_nstep_sql_td_error`` (soft Q-learning,
:1175-1245) and ``q_v_1step_td_error`` (the discrete SAC critic, :161-219).

CPU (``-m "not gpu"``):
  * the fixtures in ``tests/golden/soft_td/`` hold the seeded inputs, and the live reference reproduces their outputs;
  * every public call marshals against the ctypes prototypes (recording stand-in of test_reference_suite.py);
  * the shape assertions and error types match the reference's;
  * the reference's own ``test_q_nstep_sql_td`` and ``test_fn_m_q_1step_td_error`` run against the reference and the
    stand-in.
GPU: every output and the gradient of q, for a unit upstream gradient and for a mix on the loss and td_error_per_sample,
against the fixtures (minted from the unmodified reference by ``tests/golden/make_soft_td_golden.py``) and against the live
reference from ``oracle/_ref`` on CUDA tensors, at 1e-5 with gradients scaled by their largest magnitude; and the policy
lines of MDQN, SQL and discrete SAC before and after ``install()``.
"""
import contextlib
import glob
import json
import os

import numpy as np
import pytest
import torch
import torch.nn as nn

import di_engine_b200 as b2
from di_engine_b200 import ops
from oracle import ref_loader
from tests.test_reference_suite import _RecordingLib

HAVE_REF = ref_loader.available()
GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'soft_td')
FIELDS = {
    'mdqn': ('q', 'target_q', 'next_q', 'act', 'reward', 'done', 'weight'),
    'sql': ('q', 'next_n_q', 'action', 'next_n_action', 'reward', 'done', 'weight'),
    'qv': ('q', 'v', 'act', 'reward', 'done', 'weight'),
}
OUTS = {'mdqn': ('loss', 'per', 'gap', 'clip'), 'sql': ('loss', 'per', 'rec'), 'qv': ('loss', 'per')}
GRAD_MIX = 1.3  # upstream gradient of the loss; td_error_per_sample gets the input's 'mix'


class Quartic(nn.Module):
    """a criterion the kernel does not know: runs as torch ops on the kernel's target"""
    reduction = 'none'

    def forward(self, a, b):
        return 0.25 * (a - b) ** 4 + (a - b).abs()


CRITERIA = {
    'mse': lambda: nn.MSELoss(reduction='none'),
    'l1': lambda: nn.L1Loss(reduction='none'),
    'smoothl1': lambda: nn.SmoothL1Loss(reduction='none', beta=0.7),
    'huber': lambda: nn.HuberLoss(reduction='none', delta=0.6),
    'quartic': Quartic,
}


def _case(fn, seed, B, N, nstep=1, A=0, done='randn', weight=True, crit='mse', gamma=0.97, tau=0.03, alpha=0.9, cum=0,
          vg=None, rows=None):
    """cum: 0 off, 1 a (B,) reward, K > 1 a (K, B) reward (the reference's own test passes one); rows: 'grid' (target_q on a
    0.25 grid: log_pi[a] hits -1 / 1 exactly), 'ties' (top-1 == top-2 in half of the rows), 'inf' (next_n_q rows holding
    +inf, -inf, both and NaN)"""
    return dict(fn=fn, seed=seed, B=B, N=N, nstep=nstep, A=A, done=done, weight=weight, crit=crit, gamma=gamma, tau=tau,
                alpha=alpha, cum=cum, vg=vg, rows=rows)


def td_shape(c):
    if c['fn'] == 'qv' and c['A']:
        return (c['B'], c['A'])
    if c['fn'] == 'sql' and c['cum'] > 1:
        return (c['cum'], c['B'])
    return (c['B'], )


def make_inputs(c):
    g = torch.Generator().manual_seed(c['seed'])
    B, N = c['B'], c['N']
    lead = (B, c['A']) if c['A'] else (B, )

    def randn(*s):
        return torch.randn(*s, generator=g)

    if c['done'] == 'randn':  # the reference's own tests (tests/test_td.py:436, :598)
        done = randn(B)
    elif c['done'] == '01':
        done = torch.randint(0, 2, (B, ), generator=g).float()
    else:
        done = torch.randint(0, 2, (B, ), generator=g)
    t = {}
    if c['fn'] == 'mdqn':
        t['q'] = randn(B, N)
        if c['rows'] in ('grid', 'ties'):
            # distinct entries at least 0.5 apart from the row's max (tau > 0) or min (tau < 0): with |tau| = 1/256 every other
            # exp((x - m) / tau) underflows to 0, logsumexp is exact and log_pi[a] = x_a - x_max (tau > 0) or x_a - x_min
            # (tau < 0) exactly -- -1 and 1 are reached with x_a - x_max = -1 / x_a - x_min = 1
            off = torch.tensor([0.0, -0.5, -1.0, -1.25, -1.75, -2.25, -2.75, -3.25])[:N]
            rows = torch.stack([off[torch.randperm(N, generator=g)] for _ in range(B)])
            if c['rows'] == 'ties':  # half the rows hold their max twice
                k = torch.arange(B) % 2 == 0
                second = rows.argsort(1, descending=True)[:, 1]
                rows[k, second[k]] = 0.0
            t['target_q'] = rows + torch.randint(-3, 4, (B, 1), generator=g).float()
        else:
            t['target_q'] = randn(B, N)
        t['next_q'] = randn(B, N)
        t['act'] = torch.randint(0, N, (B, ), generator=g)
        t['reward'] = randn(B)
    elif c['fn'] == 'sql':
        t['q'] = randn(B, N)
        nq = randn(B, N) * 3
        if c['rows'] == 'inf':
            inf = float('inf')
            nq[0, 0] = inf                 # +inf -> 20
            nq[1 % B, :] = -inf            # all -inf -> -20
            nq[2 % B, 0], nq[2 % B, 1] = inf, -inf  # both -> +20
            nq[3 % B, 1] = float('nan')    # NaN stays NaN
        t['next_n_q'] = nq
        t['action'] = torch.randint(0, N, (B, ), generator=g)
        t['next_n_action'] = torch.randint(0, N, (B, ), generator=g)
        if c['cum'] == 1:
            t['reward'] = torch.rand(B, generator=g)
        else:
            t['reward'] = torch.rand(c['cum'] if c['cum'] > 1 else c['nstep'], B, generator=g)
    else:
        t['q'] = randn(*lead, N)
        t['v'] = randn(*lead)
        t['act'] = torch.randint(0, N, lead, generator=g)
        t['reward'] = randn(B)
    t['done'] = done
    t['weight'] = torch.rand(*(lead if c['fn'] == 'qv' else (B, )), generator=g) + 0.5 if c['weight'] else None
    t['mix'] = torch.linspace(-1.0, 1.5, int(np.prod(td_shape(c)))).reshape(td_shape(c))
    return t


def value_gamma_of(c):
    if c['vg'] is None:
        return None
    if c['vg'] == 'float':
        return 0.9
    if c['vg'] == '0dim':
        return torch.tensor(0.85)
    return torch.rand(c['B'], generator=torch.Generator().manual_seed(c['seed'] + 7)) * 0.2 + 0.8


# fixture cases (tests/golden/soft_td/<name>.npz)
CASES = {
    # Munchausen DQN: Atari B = 32, CartPole B = 64 (entropy_tau 0.03, m_alpha 0.9)
    'mdqn_atari': _case('mdqn', 1, 32, 6, weight=False),
    'mdqn_cartpole': _case('mdqn', 2, 64, 2, done='01'),
    'mdqn_b1': _case('mdqn', 3, 1, 2),
    'mdqn_n18_int_done': _case('mdqn', 4, 33, 18, done='int', tau=0.1, alpha=0.6),
    'mdqn_clip_lo': _case('mdqn', 5, 64, 6, rows='grid', tau=1 / 256),
    'mdqn_clip_hi': _case('mdqn', 6, 64, 6, rows='grid', tau=-1 / 256, done='01'),
    'mdqn_ties': _case('mdqn', 7, 32, 5, rows='ties', tau=1 / 256),
    'mdqn_l1': _case('mdqn', 8, 32, 6, crit='l1'),
    'mdqn_huber': _case('mdqn', 9, 32, 6, crit='huber', done='01'),
    'mdqn_custom': _case('mdqn', 10, 16, 4, crit='quartic'),
    # soft Q-learning: CartPole / LunarLander B = 64, nstep 1
    'sql_cartpole': _case('sql', 11, 64, 2, weight=False, alpha=0.12),
    'sql_lunar': _case('sql', 12, 64, 4, alpha=0.08, done='01'),
    'sql_nstep5_vg_vec': _case('sql', 13, 32, 6, 5, vg='vec'),
    'sql_nstep10_vg_0dim': _case('sql', 14, 17, 3, 10, vg='0dim', done='int'),
    'sql_vg_float': _case('sql', 15, 32, 6, 3, vg='float'),
    'sql_cum': _case('sql', 16, 32, 6, 3, cum=1),
    'sql_cum_vg_0dim': _case('sql', 17, 32, 6, 3, cum=1, vg='0dim', weight=False),
    'sql_cum_k3': _case('sql', 18, 8, 3, 3, cum=3, weight=False, alpha=0.5),
    'sql_cum_k4_vg_vec': _case('sql', 19, 8, 3, 2, cum=4, vg='vec'),
    'sql_inf': _case('sql', 20, 8, 4, 2, rows='inf', alpha=0.5),
    'sql_smoothl1': _case('sql', 21, 32, 6, 2, crit='smoothl1'),
    'sql_custom': _case('sql', 22, 16, 5, 3, crit='quartic', vg='vec'),
    # discrete SAC critic: B = 64 - 256, twin critic
    'qv_sac': _case('qv', 23, 256, 6),
    'qv_noweight': _case('qv', 24, 64, 6, weight=False, done='01'),
    'qv_int_done': _case('qv', 25, 32, 4, done='int'),
    'qv_multi': _case('qv', 26, 16, 5, A=3, weight=False),
    'qv_multi_weight': _case('qv', 27, 16, 5, A=3, done='01'),
    'qv_huber': _case('qv', 28, 64, 6, crit='huber'),
    'qv_custom': _case('qv', 29, 16, 4, A=2, crit='quartic'),
}


def run(api, c, t, dev, grad='mix'):
    """call the public function of ``api`` (the reference or ours) on case ``c``; -> dict of numpy outputs + grad_q"""
    d = {k: (v.to(dev) if isinstance(v, torch.Tensor) else v) for k, v in t.items()}
    q = d['q'].clone().requires_grad_(True)
    ops_ = [q] + [d[k] for k in FIELDS[c['fn']][1:]]
    crit = CRITERIA[c['crit']]()
    if c['fn'] == 'mdqn':
        out = api.m_q_1step_td_error(api.m_q_1step_td_data(*ops_), c['gamma'], c['tau'], c['alpha'], crit)
    elif c['fn'] == 'sql':
        vg = value_gamma_of(c)
        if isinstance(vg, torch.Tensor):
            vg = vg.to(dev)
        out = api.q_nstep_sql_td_error(api.q_nstep_td_data(*ops_), c['gamma'], c['alpha'], nstep=c['nstep'],
                                       cum_reward=bool(c['cum']), value_gamma=vg, criterion=crit)
    else:
        out = api.q_v_1step_td_error(api.q_v_1step_td_data(*ops_), c['gamma'], crit)
    res = dict(zip(OUTS[c['fn']], out))
    if grad == 'unit':
        res['loss'].backward()
    else:
        (GRAD_MIX * res['loss'] + (res['per'] * d['mix']).sum()).backward()
    res = {k: v.detach().cpu().numpy().astype(np.float64) for k, v in res.items()}
    res['grad_q'] = q.grad.detach().cpu().numpy().astype(np.float64)
    return res


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
    t = {k: (torch.from_numpy(d['in_' + k]) if 'in_' + k in d else None) for k in FIELDS[case['fn']] + ('mix', )}
    want = {k: d['out_' + k] for k in OUTS[case['fn']] + ('grad_q', )}
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
    for k in FIELDS[case['fn']] + ('mix', ):
        if want[k] is None:
            assert t[k] is None, k
        else:
            assert t[k].dtype == want[k].dtype and np.array_equal(t[k].numpy(), want[k].numpy(), equal_nan=True), k


@pytest.mark.skipif(not HAVE_REF, reason='reference not importable here')
@pytest.mark.parametrize('name', sorted(CASES))
def test_fixture_outputs_are_the_live_reference(name):
    case, t, want = load_fixture(name)
    got = run(ref_loader.load(), case, t, 'cpu')
    for k in want:
        assert np.array_equal(got[k], want[k], equal_nan=True), (name, k)


def test_fixtures_cover_the_edges():
    """the boundary cases hold what their names say, in the stored reference outputs"""
    _, t, want = load_fixture('mdqn_clip_lo')
    lp = (t['target_q'] - t['target_q'].max(1, keepdim=True)[0]).gather(1, t['act'].reshape(-1, 1)).reshape(-1)
    assert (lp == -1).any() and (lp < -1).any() and (lp > -1).any()
    assert np.array_equal(want['clip'].reshape(-1), (lp < -1).numpy().astype(np.float64))
    _, t, want = load_fixture('mdqn_clip_hi')
    lp = (t['target_q'] - t['target_q'].min(1, keepdim=True)[0]).gather(1, t['act'].reshape(-1, 1)).reshape(-1)
    assert (lp == 1).any() and (lp > 1).any() and (lp < 1).any()
    assert np.array_equal(want['clip'].reshape(-1), (lp > 1).numpy().astype(np.float64))
    _, t, want = load_fixture('mdqn_ties')
    top = t['target_q'].topk(2, 1)[0]
    assert (top[:, 0] == top[:, 1]).sum() == t['target_q'].shape[0] // 2
    _, _, want = load_fixture('sql_inf')
    assert list(want['rec'][:3]) == [20.0, -20.0, 20.0] and np.isnan(want['rec'][3])


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
    yield calls
    ops._CONST.clear()


@pytest.mark.filterwarnings('ignore:invalid value encountered in cast')  # the stand-in leaves outputs uninitialised
@pytest.mark.filterwarnings('ignore:Using a target size')
@pytest.mark.parametrize('name', sorted(CASES))
def test_marshalling_dry_run(dry, name):
    case = CASES[name]
    res = run(b2.rl_utils, case, make_inputs(case), 'cpu')
    # a custom criterion runs as torch ops around the kernel's detached target: no backward launch
    assert dry == ['b200rl_soft_td_fwd'] + ([] if case['crit'] == 'quartic' else ['b200rl_qntd_bwd']), dry
    shape = td_shape(case)
    assert res['loss'].shape == () and res['per'].shape == shape
    N = case['N']
    assert res['grad_q'].shape == ((case['B'], case['A'], N) if case['A'] else (case['B'], N))
    if case['fn'] == 'mdqn':
        assert res['gap'].shape == () and res['clip'].shape == (case['B'], 1)
    if case['fn'] == 'sql':
        assert res['rec'].shape == (case['B'], )


def _apis():
    return [b2.rl_utils] + ([ref_loader.load()] if HAVE_REF else [])


def test_error_behaviour_matches_reference(dry):
    c = CASES['mdqn_atari']
    t = make_inputs(c)
    B = c['B']
    for api in _apis():
        data = api.m_q_1step_td_data(*[t[k] for k in FIELDS['mdqn']])
        with pytest.raises(AssertionError):  # td.py:121
            api.m_q_1step_td_error(data._replace(act=t['act'].reshape(B, 1)), 0.99, 0.03, 0.9)
        with pytest.raises(AssertionError):  # td.py:122
            api.m_q_1step_td_error(data._replace(reward=t['reward'].reshape(1, B)), 0.99, 0.03, 0.9)
        with pytest.raises(RuntimeError, match='bool'):  # 1 - done, td.py:145
            api.m_q_1step_td_error(data._replace(done=t['done'] > 0), 0.99, 0.03, 0.9)
        one = torch.randn(B, 1)
        with pytest.raises(RuntimeError, match='out of range'):  # topk(2) of one action, td.py:152
            api.m_q_1step_td_error(data._replace(q=one, target_q=one, next_q=one, act=torch.zeros(B, dtype=torch.long)),
                                   0.99, 0.03, 0.9)
    c = CASES['sql_nstep5_vg_vec']
    t = make_inputs(c)
    for api in _apis():
        data = api.q_nstep_td_data(*[t[k] for k in FIELDS['sql']])
        with pytest.raises(AssertionError):  # td.py:1220
            api.q_nstep_sql_td_error(data._replace(action=t['action'].reshape(-1, 1)), 0.9, 0.5, nstep=5)
        with pytest.raises(AssertionError):  # td.py:257 through nstep_return
            api.q_nstep_sql_td_error(data, 0.9, 0.5, nstep=4)
        with pytest.raises(TypeError, match='gamma should be float or list'):  # td.py:284
            api.q_nstep_sql_td_error(data, 1, 0.5, nstep=5)
        with pytest.raises(RuntimeError, match='bool'):  # nstep_return's 1 - done, td.py:267
            api.q_nstep_sql_td_error(data._replace(done=t['done'] > 0), 0.9, 0.5, nstep=5)
    with pytest.raises(NotImplementedError):  # list gamma: DESIGN section 4
        b2.q_nstep_sql_td_error(b2.q_nstep_td_data(*[t[k] for k in FIELDS['sql']]), [torch.tensor(0.9)] * c['B'], 0.5,
                                nstep=5)
    c = CASES['qv_multi']
    t = make_inputs(c)
    for api in _apis():
        data = api.q_v_1step_td_data(*[t[k] for k in FIELDS['qv']])
        with pytest.raises(AssertionError):  # td.py:207
            api.q_v_1step_td_error(data._replace(reward=t['reward'].reshape(1, -1)), 0.9)
        with pytest.raises(AssertionError):  # td.py:200
            api.q_v_1step_td_error(data._replace(q=t['q'][:, 0], v=t['v'][:, 0], act=t['act'][:, 0],
                                                 reward=t['reward'].reshape(1, -1)), 0.9)
        with pytest.raises(RuntimeError, match='bool'):  # td.py:217
            api.q_v_1step_td_error(data._replace(done=t['done'] > 0), 0.9)


def test_cum_reward_integer_gamma_like_reference(dry):
    """with cum_reward the reference never reaches nstep_return, so an int gamma is accepted (td.py:1239)"""
    c = CASES['sql_cum']
    t = make_inputs(c)
    for api in _apis():
        api.q_nstep_sql_td_error(api.q_nstep_td_data(*[t[k] for k in FIELDS['sql']]), 1, 0.5, nstep=3, cum_reward=True)


# ---- the reference's own tests, ding/rl_utils/tests/test_td.py::test_q_nstep_sql_td (:432) and ::test_fn_m_q_1step_td_error
# (:592), seeded, in three implementations -------------------------------------------------------------------------------
PORT_FILE = os.path.join(GOLDEN_DIR, 'ported_reference_tests.npz')


def ported_body(api, dev, check_values=True):
    """check_values=False: the recording stand-in computes nothing, so only the shape assertions apply"""
    rec = {}
    g = torch.Generator().manual_seed(432)
    batch_size, action_dim = 4, 3
    next_q = torch.randn(batch_size, action_dim, generator=g).to(dev)
    done = torch.randn(batch_size, generator=g).to(dev)
    action = torch.randint(0, action_dim, size=(batch_size, ), generator=g).to(dev)
    next_action = torch.randint(0, action_dim, size=(batch_size, ), generator=g).to(dev)
    for nstep in range(1, 10):
        q = torch.randn(batch_size, action_dim, generator=g).to(dev).requires_grad_(True)
        reward = torch.rand(nstep, batch_size, generator=g).to(dev)
        data = api.q_nstep_td_data(q, next_q, action, next_action, reward, done, None)
        loss, td_error_per_sample, record_target_v = api.q_nstep_sql_td_error(data, 0.95, 1.0, nstep=nstep)
        assert td_error_per_sample.shape == (batch_size, )
        assert loss.shape == ()
        assert q.grad is None
        loss.backward()
        assert isinstance(q.grad, torch.Tensor)
        for k, v in (('sql_loss', loss), ('sql_td', td_error_per_sample), ('sql_rec', record_target_v),
                     ('sql_grad', q.grad)):
            rec['%s_%d' % (k, nstep)] = v.detach().cpu().numpy().astype(np.float64)
        data = api.q_nstep_td_data(q, next_q, action, next_action, reward, done, None)
        loss, td_error_per_sample, record_target_v = api.q_nstep_sql_td_error(data, 0.95, 0.5, nstep=nstep, cum_reward=True)
        rec['sqlcum_td_%d' % nstep] = td_error_per_sample.detach().cpu().numpy().astype(np.float64)
        value_gamma = torch.tensor(0.9).to(dev)
        data = api.q_nstep_td_data(q, next_q, action, next_action, reward, done, None)
        loss, td_error_per_sample, record_target_v = api.q_nstep_sql_td_error(
            data, 0.95, 0.5, nstep=nstep, cum_reward=True, value_gamma=value_gamma
        )
        q.grad = None
        loss.backward()
        assert isinstance(q.grad, torch.Tensor)
        rec['sqlcumvg_loss_%d' % nstep] = loss.detach().cpu().numpy().astype(np.float64)
        rec['sqlcumvg_grad_%d' % nstep] = q.grad.cpu().numpy().astype(np.float64)
    g = torch.Generator().manual_seed(592)
    batch_size, action_dim = 128, 9
    q = torch.randn(batch_size, action_dim, generator=g).to(dev).requires_grad_(True)
    target_q_current = torch.randn(batch_size, action_dim, generator=g).to(dev).requires_grad_(False)
    target_q_next = torch.randn(batch_size, action_dim, generator=g).to(dev).requires_grad_(False)
    done = torch.randn(batch_size, generator=g).to(dev)
    action = torch.randint(0, action_dim, size=(batch_size, ), generator=g).to(dev)
    reward = torch.randn(batch_size, generator=g).to(dev)
    data = api.m_q_1step_td_data(q, target_q_current, target_q_next, action, reward, done, None)
    loss, td_error_per_sample, action_gap, clip_frac = api.m_q_1step_td_error(data, 0.99, 0.03, 0.6)
    assert loss.shape == ()
    assert q.grad is None
    loss.backward()
    assert isinstance(q.grad, torch.Tensor)
    assert not check_values or clip_frac.mean().item() <= 1
    assert td_error_per_sample.shape == (batch_size, )
    for k, v in (('mdqn_loss', loss), ('mdqn_td', td_error_per_sample), ('mdqn_gap', action_gap), ('mdqn_clip', clip_frac),
                 ('mdqn_grad', q.grad)):
        rec[k] = v.detach().cpu().numpy().astype(np.float64)
    return rec


def _stored_port():
    with np.load(PORT_FILE) as z:
        return {k: z[k] for k in z.files}


@pytest.mark.filterwarnings('ignore:Using a target size')
@pytest.mark.filterwarnings('ignore:Implicit dimension choice')
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
        assert float(want['mdqn_gap']) > 0  # the reference's `action_gap.item() > 0`
    elif impl == 'b200_dry':
        request.getfixturevalue('dry')
        ported_body(b2.rl_utils, 'cpu', check_values=False)
    else:
        got = ported_body(b2.rl_utils, 'cuda')
        compare(got, ported_body(ref_loader.load(), 'cuda') if HAVE_REF else _stored_port())
        assert float(got['mdqn_gap']) > 0


# =================================================================================================================
# GPU
# =================================================================================================================
def reference_or_skip():
    if not HAVE_REF:
        pytest.skip('reference not importable here')
    return ref_loader.load()


@pytest.mark.gpu
@pytest.mark.filterwarnings('ignore:Using a target size')
@pytest.mark.filterwarnings('ignore:Implicit dimension choice')
@pytest.mark.parametrize('name', sorted(CASES))
def test_fixture_cases(name):
    case, t, want = load_fixture(name)
    compare(run(b2.rl_utils, case, t, 'cuda'), want)
    if HAVE_REF:
        ref = ref_loader.load()
        compare(run(b2.rl_utils, case, t, 'cuda', 'unit'), run(ref, case, t, 'cuda', 'unit'))
        compare(run(b2.rl_utils, case, t, 'cuda'), run(ref, case, t, 'cuda'))


SHAPES = [(1, 2, 1), (4, 1000, 3), (32, 6, 1), (64, 2, 10), (513, 6, 7), (513, 1000, 2), (1025, 6, 1), (100003, 6, 4)]


@pytest.mark.gpu
@pytest.mark.filterwarnings('ignore:Implicit dimension choice')
@pytest.mark.parametrize('B,N,nstep', SHAPES)
@pytest.mark.parametrize('fn', ['mdqn', 'sql', 'qv'])
def test_shapes_vs_reference(fn, B, N, nstep):
    ref = reference_or_skip()
    seed = 40 + B % 97 + N + nstep
    done = ('01', 'int', 'randn')[seed % 3]
    if fn == 'mdqn':
        case = _case('mdqn', seed, B, N, done=done, weight=B % 2 == 0, tau=0.03 + 0.01 * (nstep % 3))
    elif fn == 'sql':
        case = _case('sql', seed, B, N, nstep, done=done, weight=B % 2 == 1, vg=(None, 'vec', '0dim', 'float')[nstep % 4],
                     alpha=(0.05, 0.5, 1.0)[seed % 3])
    else:
        case = _case('qv', seed, B, N, A=3 if nstep % 2 else 0, done=done, weight=B % 2 == 0)
    t = make_inputs(case)
    for grad in ('unit', 'mix'):
        compare(run(b2.rl_utils, case, t, 'cuda', grad), run(ref, case, t, 'cuda', grad))


@pytest.mark.gpu
@pytest.mark.filterwarnings('ignore:Using a target size')
@pytest.mark.parametrize('name', ['mdqn_atari', 'mdqn_custom', 'sql_cum_k3', 'sql_custom', 'qv_multi', 'qv_sac'])
def test_host_buffers(name):
    """CPU tensors in: staged to the device, results back on the host, gradient back in the host q"""
    case, t, want = load_fixture(name)
    got = run(b2.rl_utils, case, t, 'cpu')
    compare(got, want)


@pytest.mark.gpu
def test_outputs_are_device_tensors_without_gradient_where_the_reference_has_none():
    case, t, _ = load_fixture('mdqn_atari')
    d = {k: (v.cuda() if v is not None else None) for k, v in t.items()}
    q = d['q'].clone().requires_grad_(True)
    loss, per, gap, clip = b2.m_q_1step_td_error(b2.m_q_1step_td_data(q, *[d[k] for k in FIELDS['mdqn'][1:]]), 0.99, 0.03,
                                                 0.9)
    assert all(x.is_cuda for x in (loss, per, gap, clip)) and loss.requires_grad and per.requires_grad
    assert not gap.requires_grad and not clip.requires_grad and clip.dtype == torch.float32
    case, t, _ = load_fixture('sql_lunar')
    d = {k: (v.cuda() if v is not None else None) for k, v in t.items()}
    q = d['q'].clone().requires_grad_(True)
    loss, per, rec = b2.q_nstep_sql_td_error(b2.q_nstep_td_data(q, *[d[k] for k in FIELDS['sql'][1:]]), 0.99, 0.08)
    assert rec.is_cuda and not rec.requires_grad and loss.requires_grad
    loss.backward()
    assert q.grad.shape == q.shape


# ---- the policy lines, with the reference functions and after install() ------------------------------------------------
def mdqn_lines(rl, q_value, target_q_value_current, target_q_value, data, gamma, entropy_tau, m_alpha):
    """ding/policy/mdqn.py:242-249 and the priority of its return dict"""
    data_m = rl.m_q_1step_td_data(
        q_value, target_q_value_current, target_q_value, data['action'], data['reward'].squeeze(0), data['done'],
        data['weight']
    )
    loss, td_error_per_sample, action_gap, clipfrac = rl.m_q_1step_td_error(data_m, gamma, entropy_tau, m_alpha)
    loss.backward()
    return loss, td_error_per_sample.abs().tolist(), action_gap, clipfrac


def sql_lines(rl, q_value, target_q_value, target_q_action, data, gamma, alpha, nstep):
    """ding/policy/sql.py:141-148"""
    data_n = rl.q_nstep_td_data(
        q_value, target_q_value, data['action'], target_q_action, data['reward'], data['done'], data['weight']
    )
    value_gamma = data.get('value_gamma')
    loss, td_error_per_sample, record_target_v = rl.q_nstep_sql_td_error(
        data_n, gamma, alpha, nstep=nstep, value_gamma=value_gamma
    )
    record_target_v = record_target_v.mean()
    loss.backward()
    return loss, td_error_per_sample.abs().tolist(), record_target_v


def sac_lines(rl, q_value, target_value, action, reward, done, data, gamma):
    """ding/policy/sac.py:262-278, twin critic"""
    loss_dict = {}
    q_data0 = rl.q_v_1step_td_data(q_value[0], target_value, action, reward, done, data['weight'])
    loss_dict['critic_loss'], td_error_per_sample0 = rl.q_v_1step_td_error(q_data0, gamma)
    q_data1 = rl.q_v_1step_td_data(q_value[1], target_value, action, reward, done, data['weight'])
    loss_dict['twin_critic_loss'], td_error_per_sample1 = rl.q_v_1step_td_error(q_data1, gamma)
    td_error_per_sample = (td_error_per_sample0 + td_error_per_sample1) / 2
    loss_dict['critic_loss'].backward()
    loss_dict['twin_critic_loss'].backward()
    return loss_dict['critic_loss'], loss_dict['twin_critic_loss'], td_error_per_sample.abs().tolist()


def _policy_runs(rl, seed):
    g = torch.Generator().manual_seed(seed)
    dev = 'cuda'
    out = {}
    B, N = 32, 6  # M-DQN on Atari
    q = torch.randn(B, N, generator=g).to(dev).requires_grad_(True)
    data = {'action': torch.randint(0, N, (B, ), generator=g).to(dev), 'reward': torch.randn(1, B, generator=g).to(dev),
            'done': torch.randint(0, 2, (B, ), generator=g).float().to(dev),
            'weight': (torch.rand(B, generator=g) + 0.5).to(dev)}
    tqc, tqn = torch.randn(B, N, generator=g).to(dev), torch.randn(B, N, generator=g).to(dev)
    loss, prio, gap, clip = mdqn_lines(rl, q, tqc, tqn, data, 0.99, 0.03, 0.9)
    out.update(mdqn_loss=loss.item(), mdqn_prio=np.array(prio), mdqn_gap=gap.item(), mdqn_clip=clip.cpu().numpy(),
               mdqn_grad=q.grad.cpu().numpy())
    B, N = 64, 4  # SQL on LunarLander, nstep 1
    q = torch.randn(B, N, generator=g).to(dev).requires_grad_(True)
    data = {'action': torch.randint(0, N, (B, ), generator=g).to(dev), 'reward': torch.rand(1, B, generator=g).to(dev),
            'done': torch.randint(0, 2, (B, ), generator=g).float().to(dev), 'weight': None}
    tq = torch.randn(B, N, generator=g).to(dev)
    loss, prio, rec = sql_lines(rl, q, tq, tq.argmax(1), data, 0.99, 0.08, 1)
    out.update(sql_loss=loss.item(), sql_prio=np.array(prio), sql_rec=rec.item(), sql_grad=q.grad.cpu().numpy())
    B, N = 256, 6  # discrete SAC, twin critic
    q = torch.randn(2, B, N, generator=g).to(dev).requires_grad_(True)
    q_value = [q[0], q[1]]
    data = {'weight': None}
    target_value = torch.randn(B, generator=g).to(dev)
    action = torch.randint(0, N, (B, ), generator=g).to(dev)
    reward, done = torch.randn(B, generator=g).to(dev), torch.randint(0, 2, (B, ), generator=g).float().to(dev)
    l0, l1, prio = sac_lines(rl, q_value, target_value, action, reward, done, data, 0.99)
    out.update(sac_loss0=l0.item(), sac_loss1=l1.item(), sac_prio=np.array(prio), sac_grad=q.grad.cpu().numpy())
    return out


@pytest.mark.gpu
def test_policy_lines_before_and_after_install():
    ref = reference_or_skip()
    want = _policy_runs(ref, 77)
    fns = ('m_q_1step_td_error', 'q_nstep_sql_td_error', 'q_v_1step_td_error')
    try:
        b2.install()
        assert all(getattr(ref, n) is getattr(b2.rl_utils, n) for n in fns)
        got = _policy_runs(ref, 77)
    finally:
        b2.uninstall()
    assert not any(getattr(ref, n) is getattr(b2.rl_utils, n) for n in fns)
    compare(got, want)
