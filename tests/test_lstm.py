"""The layer-normalised LSTM (ding/torch_utils/network/rnn.py:131-239, lstm_type='normal', norm_type='LN') on
csrc/lstm.cu, with its GEMMs on cuBLAS: ``ops.LNLSTMFunction``, the drop-in ``di_engine_b200.torch_utils.LSTM`` and the
forward ``install()`` sets on the reference class.  The reference is loaded from the archive ``oracle/ref_scatter.py``
builds (it holds rnn.py and normalization.py).

CPU (``-m "not gpu"``):
  * the float64 restatement (tests/lstm_oracle.py) matches the reference module run in float64;
  * ``install()`` patches ``LSTM.forward`` on the reference class (a model built earlier included) and ``uninstall()``
    restores it, with a recording stand-in for the library; CPU inputs through the patched forward are bit-identical to
    the unpatched reference;
  * the drop-in and the reference load each other's ``state_dict`` and draw the same weights under one seed;
  * every ``prev_state`` form gives the reference's structure and values;
  * the fixtures in ``tests/golden/lstm/`` regenerate from their seeds.
GPU, with the reference run on the same CUDA tensors, under the accuracy rule
max|ours - fp64| <= 2 max|reference fp32 - fp64| + 1e-6 max|fp64| (fp64 = the reference module in float64): the case grid,
DRQN's 80 chained per-step calls, dropout masks, determinism, strided inputs, torch.compile(fullgraph=True), the patched
reference class, and the fixtures.
"""
import contextlib
import copy
import glob
import importlib
import json
import os
import sys

import numpy as np
import pytest
import torch

import di_engine_b200 as b2
from di_engine_b200 import _lib, ops
from di_engine_b200.torch_utils import lstm as lstm_mod
from oracle import ref_scatter
from tests import lstm_oracle

HAVE_REF = ref_scatter.available()
GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'lstm')
gpu = pytest.mark.gpu
need_ref = pytest.mark.skipif(not HAVE_REF, reason='reference archive not built')
FORMS = ('none', 'list', 'list_none', 'list_pairs', 'dict')


class _NoTreeTensor:
    """stands in for treetensor's Tensor, which rnn.py's _before_forward tests per-sample states against"""


@contextlib.contextmanager
def reference_rnn():
    with ref_scatter.network():
        sys.modules['treetensor.torch'].Tensor = _NoTreeTensor  # the archive's treetensor stub is removed on exit
        yield importlib.import_module(ref_scatter.PACKAGE + '.rnn')


def _case(seed, T, B, I, H, L, form, list_next_state):
    return dict(seed=seed, T=T, B=B, I=I, H=H, L=L, form=form, lns=list_next_state)


# every value of T {1, 2, 25, 80}, B {1, 7, 64, 320}, (I, H), L {1, 2}, state form and list_next_state appears, and every
# specialisation of the step kernels runs: K = 1 (H <= 128), 2 (H = 200), 4 (H = 512), 8 (H = 1024) and the re-reading path
# K = 0 (4H > 4096) at H = 2048 and at H = 1100, whose last 128-unit block is partial
CASES = {
    't1_b1_tiny': _case(1, 1, 1, 3, 5, 1, 'none', True),
    't2_b7_l2': _case(2, 2, 7, 64, 64, 2, 'list', True),
    't25_b64_dict': _case(3, 25, 64, 512, 512, 1, 'dict', False),
    't80_b64_list_none': _case(4, 80, 64, 512, 512, 1, 'list_none', True),
    't2_b320_h1024': _case(5, 2, 320, 128, 1024, 1, 'list_pairs', False),
    't2_b7_h2048_l2': _case(6, 2, 7, 16, 2048, 2, 'dict', True),
    't25_b320_l2': _case(7, 25, 320, 64, 64, 2, 'none', False),
    't1_b64_l2_tiny': _case(8, 1, 64, 3, 5, 2, 'list_none', False),
    't80_b7_h1024': _case(9, 80, 7, 128, 1024, 1, 'list', True),
    't25_b7_h200': _case(10, 25, 7, 32, 200, 1, 'list', False),
    't2_b5_h1100_l2': _case(14, 2, 5, 24, 1100, 2, 'none', True),
}
GOLDEN_CASES = ('tiny', 'small_l2', 'mid')
GOLDEN = {
    'tiny': _case(11, 3, 2, 3, 5, 1, 'list_none', True),
    'small_l2': _case(12, 4, 3, 8, 6, 2, 'dict', False),
    'mid': _case(13, 6, 4, 16, 24, 1, 'list', True),
}


def make_inputs(c):
    """x (T, B, I), the initial state (L, B, H) pair and the upstream gradients of y, h_T and c_T, from the seed"""
    g = torch.Generator().manual_seed(c['seed'])
    T, B, I, H, L = c['T'], c['B'], c['I'], c['H'], c['L']
    x = torch.randn(T, B, I, generator=g)
    h0, c0 = torch.randn(L, B, H, generator=g) * 0.5, torch.randn(L, B, H, generator=g) * 0.5
    gy, gh, gc = torch.randn(T, B, H, generator=g), torch.randn(L, B, H, generator=g), torch.randn(L, B, H, generator=g)
    return x, h0, c0, (gy, gh, gc)


def make_state(form, h0, c0):
    """the prev_state argument of ``form`` holding h0, c0 (None entries in 'list_none' stand for zeros at samples 1, 3...)"""
    B = h0.shape[1]
    if form == 'none':
        return None
    if form == 'dict':
        return {'h': h0, 'c': c0}
    per = [(h0[:, b:b + 1], c0[:, b:b + 1]) for b in range(B)]
    if form == 'list_pairs':
        return [list(p) for p in per]
    return [None if (form == 'list_none' and b % 2) else {'h': p[0], 'c': p[1]} for b, p in enumerate(per)]


def state_tensors(ns):
    """(h, c) (L, B, H) of a next state in either form"""
    if isinstance(ns, dict):
        return ns['h'], ns['c']
    return torch.cat([d['h'] for d in ns], 1), torch.cat([d['c'] for d in ns], 1)


def run(model, c, device, dtype=torch.float32, grads=True):
    """model's output, next state and the gradients of sum(y gy) + sum(h gh) + sum(c gc) with respect to x, the initial
    state (where the form carries one) and every parameter, as float64 numpy arrays by name"""
    x, h0, c0, (gy, gh, gc) = make_inputs(c)
    x, h0, c0 = (t.to(device, dtype).requires_grad_(grads) for t in (x, h0, c0))
    y, ns = model(x, make_state(c['form'], h0, c0), list_next_state=c['lns'])
    assert isinstance(ns, list) == c['lns']
    h, cc = state_tensors(ns)
    out = {'y': y, 'h': h, 'c': cc}
    if grads:
        model.zero_grad()
        loss = (y * gy.to(device, dtype)).sum() + (h * gh.to(device, dtype)).sum() + (cc * gc.to(device, dtype)).sum()
        loss.backward()
        out['dx'] = x.grad
        if c['form'] != 'none':
            out['dh0'], out['dc0'] = h0.grad, c0.grad
            if c['form'] == 'list_none':  # the None samples start from zeros and get no gradient
                out['dh0'], out['dc0'] = out['dh0'][:, ::2], out['dc0'][:, ::2]
        for k, p in model.named_parameters():
            out['d_' + k] = p.grad
    return {k: v.detach().double().cpu().numpy() for k, v in out.items()}


def assert_rule(ours, ref32, ref64, what=''):
    """max|ours - fp64| <= 2 max|reference fp32 - fp64| + 1e-6 max|fp64|, for every array"""
    assert sorted(ours) == sorted(ref64) == sorted(ref32), (sorted(ours), sorted(ref64))
    for k in ref64:
        d = ref64[k]
        scale = float(np.abs(d).max()) if d.size else 0.0
        bound = 2 * float(np.abs(ref32[k] - d).max(initial=0.0)) + 1e-6 * scale
        err = float(np.abs(ours[k] - d).max(initial=0.0))
        assert err <= bound, '%s %s: max |ours - fp64| = %.3e > %.3e (reference fp32: %.3e, max |fp64| %.3e)' % (
            what, k, err, bound, float(np.abs(ref32[k] - d).max(initial=0.0)), scale)


def ref_model(rnn, c, dropout=0.):
    torch.manual_seed(c['seed'] + 1000)
    return rnn.LSTM(c['I'], c['H'], c['L'], 'LN', dropout)


def ours_from(ref):
    m = b2.torch_utils.LSTM(ref.input_size, ref.hidden_size, ref.num_layers, 'LN',
                            ref.dropout.p if ref.use_dropout else 0.)
    m.load_state_dict(ref.state_dict())
    return m


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------
class _RecordingLib:

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        proto = _lib.PROTOTYPES[name]

        def fn(*args):
            assert len(args) == len(proto), (name, len(args), len(proto))
            for a, ty in zip(args, proto):
                ty.from_param(a)  # raises on a type ctypes could not marshal
            self.calls.append(name)
            return 0

        return fn


@pytest.fixture
def dry(monkeypatch):
    rec = _RecordingLib()
    monkeypatch.setattr(ops, 'lib', lambda: rec)
    monkeypatch.setattr(ops, 'require_cuda', lambda: None)
    monkeypatch.setattr(ops, 'stream_ptr', lambda: 0)
    yield rec


@need_ref
@pytest.mark.parametrize('name', ['tiny', 'small_l2'])
def test_fp64_restatement_matches_the_reference_in_fp64(name):
    c = GOLDEN[name]
    with reference_rnn() as rnn:
        ref = ref_model(rnn, c).double()
        want = run(ref, c, 'cpu', torch.float64)
    x, h0, c0, (gy, gh, gc) = make_inputs(c)
    x, h0, c0 = (t.double().requires_grad_(True) for t in (x, h0, c0))
    p = {k: v.detach().clone().requires_grad_(True) for k, v in ref.state_dict().items()}
    if c['form'] == 'list_none':
        keep = torch.arange(c['B']) % 2 == 0
        h0_, c0_ = h0 * keep[None, :, None], c0 * keep[None, :, None]
    else:
        h0_, c0_ = (h0, c0) if c['form'] != 'none' else (torch.zeros_like(h0), torch.zeros_like(c0))
    y, h, cc = lstm_oracle.forward(x, h0_, c0_, p, c['L'])
    ((y * gy.double()).sum() + (h * gh.double()).sum() + (cc * gc.double()).sum()).backward()
    got = {'y': y, 'h': h, 'c': cc, 'dx': x.grad}
    if c['form'] != 'none':
        got['dh0'], got['dc0'] = h0.grad, c0.grad
        if c['form'] == 'list_none':
            got['dh0'], got['dc0'] = h0.grad[:, ::2], c0.grad[:, ::2]
    for k, v in p.items():
        got['d_' + k] = v.grad
    assert sorted(got) == sorted(want)
    for k, v in got.items():
        np.testing.assert_allclose(v.detach().numpy(), want[k], rtol=1e-10, atol=1e-12, err_msg=k)


@need_ref
def test_install_patches_the_reference_forward_and_uninstall_restores_it(dry, monkeypatch):
    c = _case(31, 3, 2, 4, 5, 2, 'list', True)
    with reference_rnn() as rnn:
        Ref = rnn.LSTM
        forward = Ref.__dict__['forward']
        early = ref_model(rnn, c)
        try:
            done = b2.install()
            assert (ref_scatter.PACKAGE + '.rnn.LSTM', 'forward') in done
            assert Ref.__dict__['forward'].__b200_original__ is forward
            assert not [d for d in b2.install() if d[0].endswith('.LSTM')]  # a second call patches nothing
            monkeypatch.setattr(lstm_mod, 'accelerated', lambda m, inputs: True)  # CPU tensors reach the dry library
            dry.calls.clear()
            x = torch.randn(c['T'], c['B'], c['I'], requires_grad=True)
            y, ns = early(x, [None] * c['B'])
            assert y.shape == (c['T'], c['B'], c['H']) and len(ns) == c['B'] and ns[0]['h'].shape == (2, 1, c['H'])
            assert dry.calls == ['b200rl_lnlstm_step_fwd'] * (c['T'] * c['L'])
            dry.calls.clear()
            (y.sum() + ns[0]['c'].sum()).backward()
            assert dry.calls == (['b200rl_lnlstm_step_bwd'] * c['T'] + ['b200rl_lnlstm_param_grads']) * c['L']
            assert all(p.grad is not None for p in early.parameters()) and x.grad.shape == x.shape
        finally:
            b2.uninstall()
        assert Ref.__dict__['forward'] is forward


@need_ref
@pytest.mark.parametrize('form', FORMS)
def test_cpu_inputs_through_the_patched_forward_are_the_reference_bits(dry, form):
    c = _case(32, 3, 4, 6, 5, 2, form, form != 'dict')
    with reference_rnn() as rnn:
        ref = ref_model(rnn, c)
        want = run(ref, c, 'cpu')
        try:
            b2.install()
            got = run(ref, c, 'cpu')
        finally:
            b2.uninstall()
    assert dry.calls == []
    for k in want:
        assert np.array_equal(want[k], got[k]), k


@need_ref
@pytest.mark.parametrize('L, dropout', [(1, 0.), (2, 0.1), (3, 0.)])
def test_state_dicts_load_both_ways_and_one_seed_draws_the_same_weights(L, dropout):
    with reference_rnn() as rnn:
        torch.manual_seed(5)
        ref = rnn.LSTM(7, 6, L, 'LN', dropout)
        torch.manual_seed(5)
        ours = b2.torch_utils.LSTM(7, 6, L, 'LN', dropout)
        a, b = ref.state_dict(), ours.state_dict()
        assert list(a) == list(b)
        for k in a:
            assert torch.equal(a[k], b[k]), k
        torch.manual_seed(6)
        other = rnn.LSTM(7, 6, L, 'LN', dropout)
        ours.load_state_dict(other.state_dict())
        ref.load_state_dict(ours.state_dict())
        for k, v in other.state_dict().items():
            assert torch.equal(ref.state_dict()[k], v) and torch.equal(ours.state_dict()[k], v), k
        assert [k for k, _ in ours.named_parameters()] == [k for k, _ in ref.named_parameters()]


@need_ref
@pytest.mark.parametrize('form', FORMS + ('bad_len', 'bad_type'))
@pytest.mark.parametrize('list_next_state', [True, False])
def test_state_forms_match_the_reference(form, list_next_state):
    L, B, H = 2, 4, 3
    g = torch.Generator().manual_seed(7)
    h0, c0 = torch.randn(L, B, H, generator=g), torch.randn(L, B, H, generator=g)
    x = torch.randn(5, B, 2, generator=g)
    with reference_rnn() as rnn:
        ref = rnn.LSTM(2, H, L, 'LN')
        ours = b2.torch_utils.LSTM(2, H, L, 'LN')
        if form in ('bad_len', 'bad_type'):
            state, err = ([None] * (B - 1), RuntimeError) if form == 'bad_len' else (h0, TypeError)
            for m in (ref, ours):
                with pytest.raises(err):
                    m._before_forward(x, state)
            return
        state = make_state(form, h0, c0)
        a, b = ref._before_forward(x, state), ours._before_forward(x, state)
        assert len(a) == len(b) == 2
        for u, v in zip(a, b):
            assert torch.equal(u, v)
        a, b = ref._after_forward([h0, c0], list_next_state), ours._after_forward([h0, c0], list_next_state)
    assert type(a) is type(b)
    if list_next_state:
        assert len(a) == len(b) == B
        for u, v in zip(a, b):
            assert list(u) == list(v) == ['h', 'c'] and all(torch.equal(u[k], v[k]) for k in u)
    else:
        assert list(a) == list(b) == ['h', 'c'] and all(torch.equal(a[k], b[k]) for k in a)


def test_drop_in_rejects_what_the_kernels_do_not_compute():
    with pytest.raises(NotImplementedError):
        b2.torch_utils.LSTM(3, 4, 1, 'BN')
    m = b2.torch_utils.LSTM(3, 4, 1, 'LN')
    with pytest.raises(TypeError):
        m(torch.randn(2, 2, 3), None)


def test_fixtures_cover_every_golden_case():
    assert sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN_DIR, '*.npz'))) == sorted(GOLDEN_CASES)


def input_sums(c):
    x, h0, c0, gs = make_inputs(c)
    return np.array([float(t.double().sum()) for t in (x, h0, c0) + gs])


@pytest.mark.parametrize('name', GOLDEN_CASES)
def test_fixture_inputs_are_the_seeded_ones(name):
    z = np.load(os.path.join(GOLDEN_DIR, name + '.npz'))
    assert json.loads(str(z['case'])) == GOLDEN[name]
    assert np.array_equal(input_sums(GOLDEN[name]), z['in_sums'])
    torch.manual_seed(GOLDEN[name]['seed'] + 1000)
    m = b2.torch_utils.LSTM(GOLDEN[name]['I'], GOLDEN[name]['H'], GOLDEN[name]['L'], 'LN')
    assert np.array_equal(np.array([float(v.double().sum()) for v in m.state_dict().values()]), z['w_sums'])


@need_ref
@pytest.mark.parametrize('name', GOLDEN_CASES)
def test_fixture_results_regenerate_from_the_reference(name):
    """the reference run again on the CPU gives the stored outputs and gradients; the tolerance only allows for another
    CPU's fp32 GEMM kernels"""
    z = np.load(os.path.join(GOLDEN_DIR, name + '.npz'))
    c = GOLDEN[name]
    with reference_rnn() as rnn:
        got = run(ref_model(rnn, c), c, 'cpu')
    assert sorted('ref_' + k for k in got) == sorted(k for k in z.files if k.startswith('ref_'))
    for k, v in got.items():
        want = z['ref_' + k].astype(np.float64)
        np.testing.assert_allclose(v, want, rtol=1e-5, atol=1e-6 * max(1.0, float(np.abs(want).max())), err_msg=k)


def test_zero_time_steps_raise_before_any_launch(dry):
    x, h, c = torch.zeros(0, 2, 3), torch.zeros(2, 4), torch.zeros(2, 4)
    w = [torch.zeros(3, 16), torch.zeros(4, 16)] + [torch.zeros(16)] * 5
    with pytest.raises(ValueError):
        ops.lnlstm_fwd_(x, h, c, *w, True)
    assert dry.calls == []


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def three_runs(c, dropout=0.):
    """(ours, reference fp32, reference fp64), all on CUDA tensors"""
    with reference_rnn() as rnn:
        ref = ref_model(rnn, c, dropout).cuda()
        ours = ours_from(ref).cuda()
        ref64 = copy.deepcopy(ref).double()
        return run(ours, c, 'cuda'), run(ref, c, 'cuda'), run(ref64, c, 'cuda', torch.float64)


@gpu
@need_ref
@pytest.mark.parametrize('name', sorted(CASES))
def test_gpu_accuracy_rule(name):
    assert_rule(*three_runs(CASES[name]), what=name)


@gpu
@need_ref
@pytest.mark.parametrize('form', FORMS)
@pytest.mark.parametrize('list_next_state', [True, False])
def test_gpu_every_state_form(form, list_next_state):
    assert_rule(*three_runs(_case(41, 3, 5, 8, 16, 2, form, list_next_state)), what=form)


class Looped(torch.nn.Module):
    """a recurrent model's learner loop (q_learning.py:1031): one call per step, the list next state chained into the
    next call"""

    def __init__(self, rnn):
        super().__init__()
        self.rnn = rnn

    def forward(self, x, prev_state):
        outs = []
        for t in range(x.shape[0]):
            y, prev_state = self.rnn(x[t:t + 1], prev_state)
            outs.append(y)
        return torch.cat(outs, 0), prev_state


def run_looped(model, x, state, gy, gh, gc):
    """outputs and every gradient of 80 chained per-step calls, a loss on every output"""
    x = x.clone().requires_grad_(True)
    h0 = state[0].clone().requires_grad_(True)
    c0 = state[1].clone().requires_grad_(True)
    B = x.shape[1]
    prev = [{'h': h0[:, b:b + 1], 'c': c0[:, b:b + 1]} for b in range(B)]
    model.zero_grad()
    y, ns = model(x, prev)
    h, c = state_tensors(ns)
    ((y * gy).sum() + (h * gh).sum() + (c * gc).sum()).backward()
    out = {'y': y, 'h': h, 'c': c, 'dx': x.grad, 'dh0': h0.grad, 'dc0': c0.grad}
    for i, p in enumerate(model.parameters()):  # by position: a compiled module prefixes the names
        out['d_%d' % i] = p.grad
    return {k: v.detach().double().cpu().numpy() for k, v in out.items()}


def looped_case(T=80, B=16, I=64, H=128, L=1, seed=51):
    c = _case(seed, T, B, I, H, L, 'list', True)
    x, h0, c0, (gy, gh, gc) = make_inputs(c)
    return c, [t.cuda() for t in (x, h0, c0, gy, gh, gc)]


@gpu
@need_ref
def test_gpu_drqn_learner_pattern_80_chained_calls():
    c, (x, h0, c0, gy, gh, gc) = looped_case()
    with reference_rnn() as rnn:
        ref = ref_model(rnn, c).cuda()
        ours = ours_from(ref).cuda()
        ref64 = copy.deepcopy(ref).double()
        res = [run_looped(Looped(m), x.to(dt), (h0.to(dt), c0.to(dt)), gy.to(dt), gh.to(dt), gc.to(dt))
               for m, dt in ((ours, torch.float32), (ref, torch.float32), (ref64, torch.float64))]
    assert_rule(*res, what='drqn')


@gpu
@need_ref
def test_gpu_patched_reference_class_through_install():
    c, (x, h0, c0, gy, gh, gc) = looped_case(T=20, B=8, seed=52)
    with reference_rnn() as rnn:
        ref = Looped(ref_model(rnn, c).cuda())
        ref64 = copy.deepcopy(ref).double()
        before = run_looped(ref, x, (h0, c0), gy, gh, gc)
        want = run_looped(ref64, x.double(), (h0.double(), c0.double()), gy.double(), gh.double(), gc.double())
        try:
            done = b2.install()
            assert (ref_scatter.PACKAGE + '.rnn.LSTM', 'forward') in done
            after = run_looped(ref, x, (h0, c0), gy, gh, gc)
        finally:
            b2.uninstall()
    assert_rule(after, before, want, what='install')
    assert any(not np.array_equal(after[k], before[k]) for k in after)  # the kernels ran, not the reference again


@gpu
@need_ref
def test_gpu_dropout_draws_the_reference_masks():
    c = _case(61, 6, 8, 16, 32, 2, 'none', False)
    with reference_rnn() as rnn:
        ref = ref_model(rnn, c, dropout=0.1).cuda().train()
        ours = ours_from(ref).cuda().train()
        torch.manual_seed(3)
        got = run(ours, c, 'cuda')
        torch.manual_seed(3)
        want = run(ref, c, 'cuda')
    for k in want:
        np.testing.assert_allclose(got[k], want[k], rtol=1e-4, atol=1e-4 * max(1.0, float(np.abs(want[k]).max())),
                                   err_msg=k)


@gpu
@need_ref
def test_gpu_two_runs_are_bit_identical():
    c = CASES['t25_b64_dict']
    with reference_rnn() as rnn:
        ours = ours_from(ref_model(rnn, c)).cuda()
    a, b = run(ours, c, 'cuda'), run(ours, c, 'cuda')
    for k in a:
        assert np.array_equal(a[k], b[k]), k


@gpu
@need_ref
def test_gpu_strided_inputs_and_states():
    c = _case(71, 5, 6, 24, 40, 2, 'dict', False)
    x, h0, c0, (gy, gh, gc) = make_inputs(c)
    T, B, I, H, L = c['T'], c['B'], c['I'], c['H'], c['L']

    def go(model, dt):
        xb = torch.zeros(B, T, 2 * I, dtype=dt, device='cuda')
        xb[:, :, ::2] = x.transpose(0, 1).to(dt)
        hb = torch.zeros(L, H, 3 * B, dtype=dt, device='cuda')
        hb[:, :, ::3] = h0.transpose(1, 2).to(dt)
        cb = torch.zeros(L, 2 * B, H, dtype=dt, device='cuda')
        cb[:, ::2] = c0.to(dt)
        xb.requires_grad_(True), hb.requires_grad_(True), cb.requires_grad_(True)
        xs, hs, cs = xb[:, :, ::2].transpose(0, 1), hb[:, :, ::3].transpose(1, 2), cb[:, ::2]
        assert not (xs.is_contiguous() or hs.is_contiguous() or cs.is_contiguous())
        model.zero_grad()
        y, ns = model(xs, {'h': hs, 'c': cs}, list_next_state=False)
        ((y * gy.to('cuda', dt)).sum() + (ns['h'] * gh.to('cuda', dt)).sum() +
         (ns['c'] * gc.to('cuda', dt)).sum()).backward()
        out = {'y': y, 'h': ns['h'], 'c': ns['c'], 'dx': xb.grad[:, :, ::2], 'dh0': hb.grad[:, :, ::3],
               'dc0': cb.grad[:, ::2]}
        out.update({'d_' + k: p.grad for k, p in model.named_parameters()})
        return {k: v.detach().double().cpu().numpy() for k, v in out.items()}

    with reference_rnn() as rnn:
        ref = ref_model(rnn, c).cuda()
        ours = ours_from(ref).cuda()
        res = [go(ours, torch.float32), go(ref, torch.float32), go(copy.deepcopy(ref).double(), torch.float64)]
    assert_rule(*res, what='strided')


@gpu
@need_ref
def test_gpu_no_grad_saves_nothing_and_matches():
    c = _case(81, 4, 8, 16, 32, 1, 'none', False)
    x, h0, c0, _ = make_inputs(c)
    with reference_rnn() as rnn:
        ours = ours_from(ref_model(rnn, c)).cuda()
    with torch.no_grad():
        y, ns = ours(x.cuda(), None, list_next_state=False)
    assert y.grad_fn is None and ns['h'].grad_fn is None
    y2, ns2 = ours(x.cuda(), None, list_next_state=False)
    assert torch.equal(y, y2.detach()) and torch.equal(ns['c'], ns2['c'].detach())
    assert y.data_ptr() != ns['h'].data_ptr()


@gpu
@need_ref
@pytest.mark.parametrize('backend', ['aot_eager', 'inductor'])
def test_gpu_fullgraph_compile_of_the_per_step_loop_matches_eager(backend):
    c, (x, h0, c0, gy, gh, gc) = looped_case(T=5, B=4, I=16, H=32, L=2, seed=91)
    with reference_rnn() as rnn:
        ours = ours_from(ref_model(rnn, c)).cuda()
    model = Looped(ours)
    torch._dynamo.reset()
    compiled = torch.compile(model, fullgraph=True, backend=backend)
    a = run_looped(model, x, (h0, c0), gy, gh, gc)
    b = run_looped(compiled, x, (h0, c0), gy, gh, gc)
    for k in a:
        if backend == 'aot_eager':
            assert np.array_equal(a[k], b[k]), k
        else:
            np.testing.assert_allclose(b[k], a[k], rtol=1e-5, atol=1e-6 * max(1.0, float(np.abs(a[k]).max())), err_msg=k)


@gpu
@need_ref
@pytest.mark.parametrize('name', GOLDEN_CASES)
def test_gpu_matches_the_fixtures(name):
    """the fixtures hold the reference's fp32 results on the CPU, whose GEMMs round differently from the same reference on
    CUDA tensors.  Ours passes the accuracy rule with the reference error taken, per element, from whichever of the two
    references is further from fp64: the rule against the CUDA reference alone is test_gpu_accuracy_rule's; this test pins
    the results to stored numbers, so that a change of the reference or of torch cannot move both sides together."""
    c = GOLDEN[name]
    z = np.load(os.path.join(GOLDEN_DIR, name + '.npz'))
    ours, ref32, ref64 = three_runs(c)
    fixture = {k: z['ref_' + k] for k in ref64}
    worst = {k: np.where(np.abs(fixture[k] - ref64[k]) > np.abs(ref32[k] - ref64[k]), fixture[k], ref32[k]) for k in ref64}
    assert_rule(ours, worst, ref64, what=name)
