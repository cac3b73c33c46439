"""DQfD n-step TD losses (``dqfd_nstep_td_error`` / ``_with_rescale``, ding/rl_utils/td.py:870-1090) and R2D3's per-step
loop over them (``dqfd_nstep_td_error_sequence``, ding/policy/r2d3.py:322-388) on the dqfd kernels of csrc/td.cu.

CPU (``-m "not gpu"``):
  * the fp32 restatement in ``tests/dqfd_oracle.py`` is bit-exact against the live reference on every fixture case;
  * every public call marshals against the ctypes prototypes (recording stand-in of test_reference_suite.py);
  * the shape assertions and error behaviour match the reference.
GPU: every output and the gradient of q, for a unit upstream gradient and for a mix of all five outputs, against the
fixtures in ``tests/golden/dqfd/`` (minted from the unmodified reference by ``tests/golden/make_dqfd_golden.py``) and
against the live reference from ``oracle/_ref`` (the oracle where the reference is not importable), at 1e-5 with
gradients scaled by their largest magnitude.
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
from tests import dqfd_oracle as orc
from tests.test_reference_suite import _RecordingLib

HAVE_REF = ref_loader.available()
GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'dqfd')
FIELDS = ('q', 'next_n_q', 'action', 'next_n_action', 'reward', 'done', 'done_one_step', 'weight', 'new_n_q_one_step',
          'next_n_action_one_step', 'is_expert')
OUTS = ('loss', 'per', 's_n', 's_1', 's_je')


class Quartic(nn.Module):
    """a criterion the kernel does not know: runs as torch ops around the kernel's targets"""
    reduction = 'none'

    def forward(self, a, b):
        return 0.25 * (a - b) ** 4 + (a - b).abs()


def h_custom(x):
    return torch.sign(x) * (torch.sqrt(torch.abs(x) + 1) - 1) + 0.05 * x


def h_inv_custom(x):
    return torch.sign(x) * (((torch.sqrt(1 + 4 * 0.05 * (torch.abs(x) + 1 + 0.05)) - 1) / (2 * 0.05)) ** 2 - 1)


CRITERIA = {
    'mse': lambda: nn.MSELoss(reduction='none'),
    'l1': lambda: nn.L1Loss(reduction='none'),
    'smoothl1': lambda: nn.SmoothL1Loss(reduction='none', beta=0.7),
    'huber': lambda: nn.HuberLoss(reduction='none', delta=0.6),
    'quartic': Quartic,
}


def make_inputs(seed, B, N, nstep, cum=False, done='randn', weight=True, expert='mixed_float', ties=None, T=None):
    """seeded operands of dqfd_nstep_td_data; T gives the (T, B) sequence layout with reward (T, nstep, B)"""
    g = torch.Generator().manual_seed(seed)
    lead = (B, ) if T is None else (T, B)

    def flags():
        if done == 'randn':  # the reference's own test (tests/test_td.py:407-408)
            return torch.randn(*lead, generator=g)
        return torch.randint(0, 2, lead, generator=g).float()

    if ties == 'const':  # every entry of a row equal
        q = torch.randn(*lead, 1, generator=g).expand(*lead, N).contiguous()
    elif ties == 'dyadic':  # a 0.25 grid: q_a - q_j == margin exactly on many (a, j), with a < j and a > j
        q = torch.randint(0, 4, lead + (N, ), generator=g).float() * 0.25
    else:
        q = torch.randn(*lead, N, generator=g)
    t = {
        'q': q,
        'next_n_q': torch.randn(*lead, N, generator=g),
        'action': torch.randint(0, N, lead, generator=g),
        'next_n_action': torch.randint(0, N, lead, generator=g),
        'reward': (torch.rand(*lead, generator=g) if cum else
                   torch.rand(nstep, B, generator=g) if T is None else torch.rand(T, nstep, B, generator=g)),
        'done': flags(),
        'done_one_step': flags(),
        'weight': torch.rand(*lead, generator=g) + 0.5 if weight else None,
        'new_n_q_one_step': torch.randn(*lead, N, generator=g),
        'next_n_action_one_step': torch.randint(0, N, lead, generator=g),
    }
    kind, _, dtype = expert.rpartition('_')
    if kind == 'all0':
        ie = torch.zeros(lead)
    elif kind == 'all1':
        ie = torch.ones(lead)
    else:
        ie = torch.randint(0, 2, lead, generator=g).float()
    t['is_expert'] = {'float': ie, 'int': ie.long(), 'bool': ie.bool()}[dtype]
    t['mix'] = torch.linspace(-1.0, 1.5, B if T is None else T * B).reshape(lead)  # upstream gradient of td_error
    return t


def value_gamma_of(kind, B, seed):
    if kind is None:
        return None
    if kind == 'float':
        return 0.9
    if kind == '0dim':
        return torch.tensor(0.85)
    return torch.rand(B, generator=torch.Generator().manual_seed(seed + 7)) * 0.2 + 0.8


def _case(seed, B=32, N=6, nstep=3, cum=False, vg=None, done='randn', weight=True, expert='mixed_float', ties=None,
          crit='mse', rescale=False, custom_trans=False, margin=0.8, lam=(1.0, 1.0, 1.0)):
    return dict(seed=seed, B=B, N=N, nstep=nstep, cum=cum, vg=vg, done=done, weight=weight, expert=expert, ties=ties,
                crit=crit, rescale=rescale, custom_trans=custom_trans, margin=margin, lam=list(lam))


# fixture cases (tests/golden/dqfd/<name>.npz): the operand and criterion space at small shapes
CASES = {
    'dqfd_atari': _case(1, 32, 6, 3, weight=False),
    'dqfd_b1': _case(2, 1, 2, 1),
    'dqfd_b4_n18_nstep9': _case(3, 4, 18, 9, expert='mixed_int'),
    'dqfd_b513_nstep10': _case(4, 513, 6, 10, vg='vec', expert='mixed_bool'),
    'dqfd_vg_float': _case(5, 32, 6, 3, vg='float', done='01'),
    'dqfd_vg_0dim': _case(6, 32, 6, 3, vg='0dim', lam=(0.7, 0.3, 1.3)),
    'dqfd_cum': _case(7, 32, 6, 3, cum=True),
    'dqfd_cum_vg_vec': _case(8, 32, 6, 5, cum=True, vg='vec', done='01'),
    'dqfd_cum_vg_float_noweight': _case(9, 4, 3, 2, cum=True, vg='float', weight=False),
    'dqfd_all0': _case(10, 32, 6, 3, expert='all0_float'),
    'dqfd_all1_bool': _case(11, 32, 6, 3, expert='all1_bool'),
    'dqfd_l1': _case(12, 32, 6, 3, crit='l1'),
    'dqfd_smoothl1': _case(13, 32, 6, 3, crit='smoothl1', done='01'),
    'dqfd_huber': _case(14, 32, 6, 3, crit='huber'),
    'dqfd_custom_crit': _case(15, 32, 6, 3, crit='quartic', vg='vec'),
    'dqfd_custom_crit_cum': _case(16, 8, 4, 3, crit='quartic', cum=True),
    'dqfd_margin0': _case(17, 32, 6, 3, margin=0.0),
    'dqfd_ties_const': _case(18, 32, 6, 3, ties='const'),
    'dqfd_ties_const_margin0': _case(19, 32, 6, 3, ties='const', margin=0.0),
    'dqfd_ties_dyadic': _case(20, 64, 6, 3, ties='dyadic', margin=0.5, done='01'),
    'dqfd_ties_dyadic_margin025': _case(21, 64, 4, 2, ties='dyadic', margin=0.25, expert='mixed_int'),
    'dqfdr_r2d3': _case(22, 64, 6, 5, rescale=True, vg='vec', lam=(1.0, 1.0, 0.8), margin=1.0),
    'dqfdr_cum': _case(23, 32, 6, 3, rescale=True, cum=True),
    'dqfdr_huber_vg_float': _case(24, 32, 6, 9, rescale=True, crit='huber', vg='float'),
    'dqfdr_custom_trans': _case(25, 32, 6, 3, rescale=True, custom_trans=True, vg='vec'),
    'dqfdr_custom_trans_crit': _case(26, 16, 5, 3, rescale=True, custom_trans=True, crit='smoothl1', cum=True),
    'dqfdr_custom_both': _case(27, 16, 5, 4, rescale=True, custom_trans=True, crit='quartic'),
    'dqfdr_ties_dyadic': _case(28, 64, 6, 3, rescale=True, ties='dyadic', margin=0.5),
}

GRAD_MIX = (1.3, 0.7, -0.4, 1.9)  # upstream gradients of loss, s_n, s_1, s_je; td_error gets the input's 'mix'


def run(api, case, t, dev, grad='mix'):
    """call the public API of ``api`` (the reference, the oracle or ours) on ``case``; -> dict of numpy outputs + grad_q"""
    c = case
    data_t = {k: (v.to(dev) if isinstance(v, torch.Tensor) else v) for k, v in t.items()}
    q = data_t['q'].clone().requires_grad_(True)
    vg = value_gamma_of(c['vg'], c['B'], c['seed'])
    if isinstance(vg, torch.Tensor):
        vg = vg.to(dev)
    lam_n, lam_s, lam_1 = c['lam']
    crit = CRITERIA[c['crit']]()
    kw = dict(nstep=c['nstep'], cum_reward=c['cum'], value_gamma=vg, criterion=crit)
    ops_ = [q] + [data_t[k] for k in FIELDS[1:]]
    if api is orc:
        extra = {}
        if c['custom_trans']:
            extra = dict(trans_fn=h_custom, inv_trans_fn=h_inv_custom)
        loss, per, st = orc.dqfd_nstep_td_error(*ops_, c.get('gamma', 0.95), lam_n, lam_s, c['margin'], lam_1,
                                               rescale=c['rescale'], **kw, **extra)
    else:
        data = api.dqfd_nstep_td_data(*ops_)
        if c['rescale']:
            if c['custom_trans']:
                kw.update(trans_fn=h_custom, inv_trans_fn=h_inv_custom)
            loss, per, st = api.dqfd_nstep_td_error_with_rescale(data, 0.95, lam_n, lam_s, lam_1, c['margin'], **kw)
        else:
            loss, per, st = api.dqfd_nstep_td_error(data, 0.95, lam_n, lam_s, c['margin'], lam_1, **kw)
    out = {'loss': loss, 'per': per, 's_n': st[0], 's_1': st[1], 's_je': st[2]}
    if grad == 'unit':
        loss.backward()
    else:
        a, b_, c_, d_ = GRAD_MIX
        (a * loss + (per * data_t['mix']).sum() + b_ * st[0] + c_ * st[1] + d_ * st[2]).backward()
    res = {k: v.detach().cpu().numpy().astype(np.float64) for k, v in out.items()}
    res['grad_q'] = q.grad.detach().cpu().numpy().astype(np.float64)
    return res


def reference_api():
    return ref_loader.load() if HAVE_REF else orc


def compare(got, want, tol=1e-5):
    assert set(got) >= set(want), set(want) - set(got)
    for k in want:
        a, b = np.asarray(got[k], np.float64), np.asarray(want[k], np.float64)
        assert a.shape == b.shape, (k, a.shape, b.shape)
        scale = max(1.0, float(np.max(np.abs(b)))) if k.startswith('grad') and b.size else 1.0
        assert np.allclose(a, b, rtol=tol, atol=tol * scale), (k, float(np.max(np.abs(a - b))))


def load_fixture(name):
    with np.load(os.path.join(GOLDEN_DIR, name + '.npz'), allow_pickle=False) as z:
        d = {k: z[k] for k in z.files}
    case = json.loads(str(d.pop('case')))
    t = {}
    for k in FIELDS + ('mix', ):
        if 'in_' + k in d:
            t[k] = torch.from_numpy(d['in_' + k])
        else:
            t[k] = None
    want = {k: d['out_' + k] for k in OUTS + ('grad_q', )}
    return case, t, want


def fixture_names():
    return sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN_DIR, 'dqfd*.npz')))


# =================================================================================================================
# CPU
# =================================================================================================================
def test_fixture_set_matches_cases():
    assert fixture_names() == sorted(CASES)


@pytest.mark.parametrize('name', sorted(CASES))
def test_fixture_inputs_are_the_seeded_case(name):
    case, t, _ = load_fixture(name)
    assert case == CASES[name]
    want = make_inputs(case['seed'], case['B'], case['N'], case['nstep'], case['cum'], case['done'], case['weight'],
                       case['expert'], case['ties'])
    for k in FIELDS + ('mix', ):
        if want[k] is None:
            assert t[k] is None, k
        else:
            assert t[k].dtype == want[k].dtype and torch.equal(t[k], want[k]), k


@pytest.mark.parametrize('name', sorted(CASES))
def test_oracle_bit_exact_vs_reference(name):
    """the restatement against the stored reference values, and against the live reference where it is importable"""
    case, t, want = load_fixture(name)
    got = run(orc, case, t, 'cpu')
    for k in want:
        assert np.array_equal(got[k], want[k]), (name, k, float(np.max(np.abs(got[k] - want[k]))))
    if HAVE_REF:
        live = run(ref_loader.load(), case, t, 'cpu')
        for k in live:
            assert np.array_equal(got[k], live[k]), (name, k)
        live_unit, got_unit = run(ref_loader.load(), case, t, 'cpu', 'unit'), run(orc, case, t, 'cpu', 'unit')
        assert np.array_equal(got_unit['grad_q'], live_unit['grad_q']), name


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
@pytest.mark.parametrize('name', sorted(CASES))
def test_marshalling_dry_run(dry, name):
    case = CASES[name]
    t = make_inputs(case['seed'], case['B'], case['N'], case['nstep'], case['cum'], case['done'], case['weight'],
                    case['expert'], case['ties'])
    res = run(b2.rl_utils, case, t, 'cpu')
    assert dry[0] == 'b200rl_dqfd_fwd' and dry[-1] == 'b200rl_dqfd_bwd', dry
    assert res['per'].shape == (case['B'], ) and res['loss'].shape == () and res['grad_q'].shape == (case['B'], case['N'])
    assert all(res[k].shape == () for k in ('s_n', 's_1', 's_je'))


def test_sequence_marshalling_dry_run(dry):
    T, B, N, nstep = 5, 8, 6, 3
    t = make_inputs(30, B, N, nstep, T=T)
    q = t['q'].clone().requires_grad_(True)
    data = b2.dqfd_nstep_td_seq_data(q, *[t[k] for k in FIELDS[1:]])
    loss, prio, td, st = b2.dqfd_nstep_td_error_sequence(data, 0.97, 1.0, 1.0, 0.8, 1.0, nstep,
                                                         value_gamma=torch.rand(T, B), rescale=True)
    (loss + td.sum() + st[2]).backward()
    assert dry == ['b200rl_dqfd_fwd', 'b200rl_dqfd_bwd']
    assert prio.shape == (B, ) and td.shape == (T, B) and q.grad.shape == (T, B, N)


def _apis():
    return [b2.rl_utils] + ([ref_loader.load()] if HAVE_REF else [])


def test_error_behaviour_matches_reference(dry):
    t = make_inputs(31, 8, 4, 3)
    for api in _apis():
        data = api.dqfd_nstep_td_data(*[t[k] for k in FIELDS])
        with pytest.raises(AssertionError):  # td.py:933
            api.dqfd_nstep_td_error(data._replace(action=torch.zeros(8, 1, dtype=torch.long)), 0.9, 1., 1., 0.8, nstep=3)
        with pytest.raises(AssertionError):  # td.py:1031
            api.dqfd_nstep_td_error_with_rescale(data._replace(action=torch.zeros(8, 1, dtype=torch.long)), 0.9, 1., 1.,
                                                 1., 0.8, nstep=3)
        with pytest.raises(AssertionError):  # td.py:257 through nstep_return
            api.dqfd_nstep_td_error(data, 0.9, 1., 1., 0.8, nstep=2)
        with pytest.raises(TypeError, match='gamma should be float or list'):  # td.py:284
            api.dqfd_nstep_td_error(data, 1, 1., 1., 0.8, nstep=3)
    data = b2.dqfd_nstep_td_data(*[t[k] for k in FIELDS])
    with pytest.raises(NotImplementedError):  # list gamma: DESIGN section 4
        b2.dqfd_nstep_td_error(data, [torch.tensor(0.9)] * 8, 1., 1., 0.8, nstep=3)
    s = make_inputs(32, 4, 3, 2, T=3)
    seq = b2.dqfd_nstep_td_seq_data(*[s[k] for k in FIELDS])
    with pytest.raises(NotImplementedError):
        b2.dqfd_nstep_td_error_sequence(seq, 0.9, 1., 1., 0.8, nstep=2, criterion=Quartic())
    with pytest.raises(AssertionError):
        b2.dqfd_nstep_td_error_sequence(seq, 0.9, 1., 1., 0.8, nstep=3)


def test_cum_reward_integer_gamma_like_reference(dry):
    """with cum_reward the reference never reaches nstep_return, so an int gamma is accepted (td.py:945, :958)"""
    t = make_inputs(33, 8, 4, 3, cum=True)
    b2.dqfd_nstep_td_error(b2.dqfd_nstep_td_data(*[t[k] for k in FIELDS]), 1, 1., 1., 0.8, nstep=3, cum_reward=True)
    if HAVE_REF:
        ref = ref_loader.load()
        ref.dqfd_nstep_td_error(ref.dqfd_nstep_td_data(*[t[k] for k in FIELDS]), 1, 1., 1., 0.8, nstep=3,
                                cum_reward=True)


# =================================================================================================================
# GPU
# =================================================================================================================
@pytest.mark.gpu
@pytest.mark.parametrize('name', sorted(CASES))
def test_fixture_cases(name):
    case, t, want = load_fixture(name)
    compare(run(b2.rl_utils, case, t, 'cuda'), want)
    compare(run(b2.rl_utils, case, t, 'cuda', 'unit'), run(reference_api(), case, t, 'cpu', 'unit'))


SHAPES = [(1, 2, 1), (4, 6, 3), (4, 1000, 10), (32, 6, 3), (32, 18, 9), (513, 6, 10), (513, 1000, 3), (100003, 6, 3),
          (100003, 18, 10)]


@pytest.mark.gpu
@pytest.mark.parametrize('B,N,nstep', SHAPES)
@pytest.mark.parametrize('rescale', [False, True])
def test_shapes_vs_reference(B, N, nstep, rescale):
    case = _case(40 + B % 97 + N + nstep, B, N, nstep, vg='vec' if nstep % 2 else None, rescale=rescale,
                 expert='mixed_int', done='01' if B > 100 else 'randn', lam=(0.9, 0.6, 1.1))
    t = make_inputs(case['seed'], B, N, nstep, done=case['done'], expert=case['expert'])
    want_api = reference_api()
    for grad in ('unit', 'mix'):
        compare(run(b2.rl_utils, case, t, 'cuda', grad), run(want_api, case, t, 'cpu', grad))


@pytest.mark.gpu
@pytest.mark.parametrize('name', ['dqfd_atari', 'dqfd_cum', 'dqfdr_custom_both', 'dqfd_ties_dyadic'])
def test_host_buffers(name):
    """CPU tensors in: staged to the device, results back on the host, gradient back in the host q"""
    case, t, want = load_fixture(name)
    got = run(b2.rl_utils, case, t, 'cpu')
    compare(got, want)


@pytest.mark.gpu
def test_loss_is_a_device_tensor_and_backward_needs_no_sync():
    case, t, _ = load_fixture('dqfd_atari')
    q = t['q'].cuda().requires_grad_(True)
    data = b2.dqfd_nstep_td_data(q, *[x.cuda() if x is not None else None for x in (t[k] for k in FIELDS[1:])])
    loss, per, st = b2.dqfd_nstep_td_error(data, 0.95, 1., 1., 0.8, nstep=3)
    assert loss.is_cuda and per.is_cuda and all(s.is_cuda and s.shape == () for s in st)
    loss.backward()
    assert q.grad.shape == q.shape


# ---- the reference's own test, ding/rl_utils/tests/test_td.py::test_dqfd_nstep_td, in three implementations ----------
PORT_FILE = os.path.join(GOLDEN_DIR, 'ported_test_dqfd_nstep_td.npz')


def ported_body(api, dev):
    g = torch.Generator().manual_seed(403)
    batch_size, action_dim = 4, 3
    next_q = torch.randn(batch_size, action_dim, generator=g).to(dev)
    done = torch.randn(batch_size, generator=g).to(dev)
    done_1 = torch.randn(batch_size, generator=g).to(dev)
    next_q_one_step = torch.randn(batch_size, action_dim, generator=g).to(dev)
    action = torch.randint(0, action_dim, size=(batch_size, ), generator=g).to(dev)
    next_action = torch.randint(0, action_dim, size=(batch_size, ), generator=g).to(dev)
    next_action_one_step = torch.randint(0, action_dim, size=(batch_size, ), generator=g).to(dev)
    is_expert = torch.ones((batch_size)).to(dev)
    rec = {}
    for nstep in range(1, 10):
        q = torch.randn(batch_size, action_dim, generator=g).to(dev).requires_grad_(True)
        reward = torch.rand(nstep, batch_size, generator=g).to(dev)
        data = api.dqfd_nstep_td_data(q, next_q, action, next_action, reward, done, done_1, None, next_q_one_step,
                                      next_action_one_step, is_expert)
        loss, td_error_per_sample, loss_statistics = api.dqfd_nstep_td_error(
            data, 0.95, lambda_n_step_td=1, lambda_supervised_loss=1, margin_function=0.8, nstep=nstep
        )
        assert td_error_per_sample.shape == (batch_size, )
        assert loss.shape == ()
        assert q.grad is None
        loss.backward()
        assert isinstance(q.grad, torch.Tensor)
        for k, v in (('loss', loss), ('td', td_error_per_sample), ('grad', q.grad), ('s_n', loss_statistics[0]),
                     ('s_1', loss_statistics[1]), ('s_je', loss_statistics[2])):
            rec['%s_%d' % (k, nstep)] = v.detach().cpu().numpy().astype(np.float64)
    return rec


def _stored_port():
    with np.load(PORT_FILE) as z:
        return {k: z[k] for k in z.files}


@pytest.mark.parametrize('impl', [
    pytest.param('reference', marks=pytest.mark.skipif(not HAVE_REF, reason='reference not importable here')),
    pytest.param('b200_dry'),
    pytest.param('b200', marks=pytest.mark.gpu),
])
def test_dqfd_nstep_td(impl, request):
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
        compare(got, ported_body(ref_loader.load(), 'cpu') if HAVE_REF else _stored_port())


# ---- the sequence form against R2D3's literal loop (ding/policy/r2d3.py:317-388) around the reference functions --------
def r2d3_loop(api, d, gamma, lambda1, lambda2, margin_function, lambda_one_step_td, nstep, value_rescale, value_gamma):
    """R2D3Policy._forward_learn from the loss on: the positional call of r2d3.py:340-370 for both branches"""
    loss, loss_nstep, loss_1step, loss_sl, td_error = [], [], [], [], []
    for t in range(d['q'].shape[0]):
        td_data = api.dqfd_nstep_td_data(*[d[k][t] for k in FIELDS])
        fn = api.dqfd_nstep_td_error_with_rescale if value_rescale else api.dqfd_nstep_td_error
        l, e, loss_statistics = fn(td_data, gamma, lambda1, lambda2, margin_function, lambda_one_step_td, nstep, False,
                                   value_gamma=value_gamma[t])
        loss.append(l)
        td_error.append(e)
        loss_nstep.append(loss_statistics[0])
        loss_1step.append(loss_statistics[1])
        loss_sl.append(loss_statistics[2])
    loss = sum(loss) / (len(loss) + 1e-8)
    stats = [sum(x) / (len(x) + 1e-8) for x in (loss_nstep, loss_1step, loss_sl)]
    prio = 0.9 * torch.max(torch.stack(td_error), dim=0)[0] + (1 - 0.9) * (
        torch.sum(torch.stack(td_error), dim=0) / (len(td_error) + 1e-8))
    return loss, prio, torch.stack(td_error), stats


def _seq_results(loss, prio, td, stats, q, mix):
    (1.3 * loss + (td * mix).sum() + 0.7 * stats[0] - 0.4 * stats[1] + 1.9 * stats[2]).backward()
    out = {'loss': loss, 'prio': prio, 'td': td, 's_n': stats[0], 's_1': stats[1], 's_je': stats[2], 'grad_q': q.grad}
    return {k: v.detach().cpu().numpy().astype(np.float64) for k, v in out.items()}


@pytest.mark.gpu
@pytest.mark.parametrize('value_rescale', [False, True])
@pytest.mark.parametrize('lams', [(1.0, 1.0, 0.8, 1.0), (0.9, 0.5, 0.8, 0.6), (1.0, -0.5, 0.8, -1.0)])
def test_sequence_vs_r2d3_loop(value_rescale, lams):
    """T = 42 - 2 - 5 = 35, B = 64, N = 6, nstep = 5 (the Pong / LunarLander configs); a negative lambda makes some
    per-step errors negative, which the priority's max and mean see as they are"""
    T, B, N, nstep, gamma = 35, 64, 6, 5, 0.997
    lambda1, lambda2, margin, lambda_one = lams
    t = make_inputs(50 + int(value_rescale), B, N, nstep, done='01', T=T)
    vg = torch.rand(T, B, generator=torch.Generator().manual_seed(51)) * 0.1 + 0.9
    api = reference_api()
    if api is orc:  # the oracle's sequence form binds by name: give it what R2D3's positional call binds
        qr = t['q'].clone().requires_grad_(True)
        m, l1 = (lambda_one, margin) if value_rescale else (margin, lambda_one)
        want = _seq_results(*orc.dqfd_nstep_td_error_sequence(qr, *[t[k] for k in FIELDS[1:]], gamma, lambda1, lambda2, m,
                                                              l1, nstep, vg, rescale=value_rescale), qr, t['mix'])
    else:
        qr = t['q'].clone().requires_grad_(True)
        d = dict(t, q=qr)
        want = _seq_results(*r2d3_loop(api, d, gamma, lambda1, lambda2, margin, lambda_one, nstep, value_rescale, vg),
                            qr, t['mix'])
    qg = t['q'].cuda().requires_grad_(True)
    data = b2.dqfd_nstep_td_seq_data(qg, *[t[k].cuda() for k in FIELDS[1:]])
    # with rescale on, R2D3's positional list binds its margin to lambda_one_step_td and the other way round
    m, l1 = (lambda_one, margin) if value_rescale else (margin, lambda_one)
    got = _seq_results(*b2.dqfd_nstep_td_error_sequence(data, gamma, lambda1, lambda2, m, l1, nstep, value_gamma=vg.cuda(),
                                                        rescale=value_rescale), qg, t['mix'].cuda())
    compare(got, want)
    if lambda_one < 0:
        assert (want['td'] < 0).any()  # the priority sees negative errors


@pytest.mark.gpu
def test_sequence_unit_gradient_and_host_buffers():
    T, B, N, nstep = 7, 33, 6, 3
    t = make_inputs(60, B, N, nstep, T=T, weight=False)
    vg = torch.rand(T, B, generator=torch.Generator().manual_seed(61)) * 0.1 + 0.9
    qr = t['q'].clone().requires_grad_(True)
    loss_r, prio_r, td_r, st_r = orc.dqfd_nstep_td_error_sequence(qr, *[t[k] for k in FIELDS[1:]], 0.99, 1.0, 1.0, 0.8,
                                                                  1.0, nstep, vg)
    loss_r.backward()
    for dev in ('cuda', 'cpu'):
        q = t['q'].clone().to(dev).requires_grad_(True)
        data = b2.dqfd_nstep_td_seq_data(q, *[t[k].to(dev) if t[k] is not None else None for k in FIELDS[1:]])
        loss, prio, td, st = b2.dqfd_nstep_td_error_sequence(data, 0.99, 1.0, 1.0, 0.8, 1.0, nstep, value_gamma=vg.to(dev))
        loss.backward()
        assert loss.device.type == dev and prio.device.type == dev
        compare({'loss': loss.detach().cpu(), 'prio': prio.cpu(), 'td': td.detach().cpu(), 'grad_q': q.grad.cpu()},
                {'loss': loss_r.detach(), 'prio': prio_r, 'td': td_r.detach(), 'grad_q': qr.grad})
