"""COMA's loss, ``coma_error`` (ding/rl_utils/coma.py:10-58), on csrc/td.cu's lambda-return scan (COMA head) and the COMA
policy head of csrc/pg.cu.

CPU (``-m "not gpu"``):
  * the fixtures in ``tests/golden/coma/`` hold seeded inputs, the three losses and all four input gradients, minted from the
    unmodified reference; the float64 restatement (tests/coma_oracle.py) agrees with them;
  * signature and namedtuple parity, the reference's errors, TypeError for fp16 / bf16 / fp64, IndexError for an
    out-of-range action under ``B200RL_CHECK_INDICES=1``;
  * every call marshals against the ctypes prototypes, one forward entry point and one verify launch backward;
  * ``install()`` / ``uninstall()`` rebind ``coma_error`` in ``ding.rl_utils``, ``ding.rl_utils.coma`` and a policy module.
GPU: the reference (from the ``oracle/_ref`` archive) on the same CUDA tensors, losses and gradients within
1e-5 + 1e-5 * |ref|, on the fixtures' cases, strided views, several upstream gradients, repeated and interleaved backward
passes and every requires_grad combination of target_q_value / reward; the fixtures; determinism; the fullgraph compile;
the ported reference test; COMAPolicy's loss block (policy/coma.py:205-218) before and after ``install()``.
"""
import contextlib
import glob
import inspect
import json
import os
import sys
import types

import numpy as np
import pytest
import torch

import di_engine_b200 as b2
from di_engine_b200 import ops
from oracle import ref_coma, ref_loader
from tests import coma_oracle as oracle
from tests.test_reference_suite import _RecordingLib

HAVE_REF = ref_coma.available()
GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'coma')
INPUTS = ('logit', 'action', 'q_value', 'target_q_value', 'reward', 'weight')
DIFF = ('logit', 'q_value', 'target_q_value', 'reward')
RECORD = (0.001, 1.0, -0.01)  # COMAPolicy's loss weights (policy/coma.py:77-81, 213-214)
UPSTREAMS = {'record': RECORD, 'ones': (1.0, 1.0, 1.0), 'mixed': (0.37, 0.0, 2.0), 'zero': (0.0, 0.0, 0.0)}
gpu = pytest.mark.gpu


def _case(seed, T, B, A, N, weight=None, mask=None, gamma=0.99, lambda_=0.95):
    """weight: None, 'rand' (rand + 1, as the reference test), 'int', 'bool', 'bcast_b' (T, B, 1), 'bcast_a' (T, 1, A);
    mask: None, 'big' (-9999999, COMAPolicy's mask) or 'inf', each with rows that keep a single legal action"""
    return dict(seed=seed, T=T, B=B, A=A, N=N, weight=weight, mask=mask, gamma=gamma, lambda_=lambda_)


CASES = {
    'ref_none': _case(1, 128, 4, 8, 32),
    'ref_weight': _case(2, 128, 4, 8, 32, 'rand'),
    'smac_3s5z': _case(3, 10, 32, 10, 18, mask='big', lambda_=0.8),
    'smac_mmm': _case(4, 20, 32, 8, 14, 'rand', mask='big', lambda_=0.8),
    'smac_2c64zg': _case(5, 20, 32, 2, 70, mask='inf', lambda_=0.8),
    'mask_big_single': _case(6, 6, 4, 3, 9, mask='big'),
    'mask_inf_single': _case(7, 6, 4, 3, 9, 'rand', mask='inf'),
    't2': _case(8, 2, 5, 3, 6),
    'n1': _case(9, 5, 3, 2, 1),
    'n257': _case(10, 4, 3, 2, 257, 'rand'),
    'w_int': _case(11, 7, 4, 3, 5, 'int'),
    'w_bool': _case(12, 7, 4, 3, 5, 'bool'),
    'w_bcast_b': _case(13, 7, 4, 3, 5, 'bcast_b'),
    'w_bcast_a': _case(14, 7, 4, 3, 5, 'bcast_a'),
}


def make_inputs(c):
    g = torch.Generator().manual_seed(c['seed'])
    T, B, A, N = c['T'], c['B'], c['A'], c['N']
    logit = torch.randn(T, B, A, N, generator=g)
    action = torch.randint(0, N, (T, B, A), generator=g)
    if c['mask'] is not None:
        legal = torch.rand(T, B, A, N, generator=g) < 0.6
        legal[0, 0, :] = False  # a single legal action
        legal.scatter_(-1, action.unsqueeze(-1), True)  # the taken action is legal (COMAPolicy samples among them)
        logit = logit.masked_fill(~legal, -9999999.0 if c['mask'] == 'big' else float('-inf'))
    w = c['weight']
    weight = None
    if w == 'rand':
        weight = torch.rand(T, B, A, generator=g) + 1
    elif w == 'int':
        weight = torch.randint(0, 3, (T, B, A), generator=g)
    elif w == 'bool':
        weight = torch.rand(T, B, A, generator=g) < 0.7
    elif w == 'bcast_b':
        weight = torch.rand(T, B, 1, generator=g) + 0.5
    elif w == 'bcast_a':
        weight = torch.rand(T, 1, A, generator=g) + 0.5
    return {'logit': logit, 'action': action, 'q_value': torch.randn(T, B, A, N, generator=g),
            'target_q_value': torch.randn(T, B, A, N, generator=g), 'reward': torch.rand(T, B, generator=g),
            'weight': weight}


def run(coma_error, data_cls, t, device, c, upstream=(1.0, 1.0, 1.0), grads=DIFF):
    """coma_error on fresh copies of ``t`` on ``device``; -> the losses and the gradients of ``grads`` (numpy, float64)"""
    x = {k: (v.to(device).clone() if v is not None else None) for k, v in t.items()}
    for k in grads:
        x[k].requires_grad_(True)
    loss = coma_error(data_cls(*(x[k] for k in INPUTS)), c['gamma'], c['lambda_'])
    out = {k: getattr(loss, k).detach().cpu().double().numpy() for k in ('policy_loss', 'q_value_loss', 'entropy_loss')}
    total = sum(u * l for u, l in zip(upstream, loss))
    if total.requires_grad:
        total.backward()
    for k in DIFF:
        gk = x[k].grad
        out['grad_' + k] = None if gk is None else gk.detach().cpu().double().numpy()
    return out


def close(want, got, what):
    want, got = np.asarray(want, np.float64), np.asarray(got, np.float64)
    assert want.shape == got.shape, (what, want.shape, got.shape)
    with np.errstate(invalid='ignore'):
        ok = (np.isnan(want) & np.isnan(got)) | (want == got) | (np.abs(got - want) <= 1e-5 + 1e-5 * np.abs(want))
    bad = np.argwhere(~ok)
    assert ok.all(), '%s: %d of %d differ, first at %s: want %r got %r' % (
        what, len(bad), ok.size, bad[0], want[tuple(bad[0])], got[tuple(bad[0])])


def compare(want, got, keys=None):
    for k in keys or want:
        if want[k] is None:
            assert got[k] is None, k
        else:
            close(want[k], got[k], k)


FULL_MAX = 4096  # a fixture stores larger gradients as a seeded sample of this many entries and their float64 sum


def sample_index(n):
    return np.sort(np.random.default_rng(n).choice(n, FULL_MAX, replace=False)) if n > FULL_MAX else None


def pack(out):
    """the fixture form of run()'s results: float32 values, large gradients sampled"""
    arrays = {}
    for k, v in out.items():
        v = np.asarray(v)
        idx = sample_index(v.size)
        arrays['out_' + k] = (v.reshape(-1)[idx] if idx is not None else v).astype(np.float32)
        if idx is not None:
            arrays['sum_' + k] = np.float64(v.sum())
    return arrays


def compare_packed(z, got, pre=''):
    """run()-style results against a fixture's packed values (a sampled gradient: its entries and its sum)"""
    for k in [f[len(pre) + 4:] for f in z.files if f.startswith(pre + 'out_')]:
        v = np.asarray(got[k])
        idx = sample_index(v.size)
        close(z[pre + 'out_' + k], v.reshape(-1)[idx] if idx is not None else v, k)
        if idx is not None:
            assert abs(v.sum() - z[pre + 'sum_' + k]) <= 1e-4 + 1e-4 * np.abs(v).sum(), k


def input_sums(t):
    return np.array([float(t[k].double().sum()) if t[k] is not None else 0.0 for k in INPUTS])


def golden(name):
    """-> (case, its seeded inputs, the fixture); the fixture holds the inputs' sums, not the inputs"""
    z = np.load(os.path.join(GOLDEN_DIR, name + '.npz'))
    c = json.loads(str(z['case']))
    return c, make_inputs(c), z


@contextlib.contextmanager
def reference():
    with ref_coma.module() as mod:
        yield mod


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------
def test_fixtures_cover_every_case():
    assert sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN_DIR, '*.npz'))) == sorted(
        list(CASES) + ['ported_reference_test'])


@pytest.mark.parametrize('name', sorted(CASES))
def test_fixture_inputs_are_the_seeded_ones(name):
    c, t, z = golden(name)
    assert c == CASES[name]
    assert np.array_equal(input_sums(t), z['in_sums'])


@pytest.mark.parametrize('name', sorted(CASES))
def test_restatement_matches_the_fixtures(name):
    c, t, z = golden(name)
    compare_packed(z, oracle.coma(*(t[k] for k in INPUTS), c['gamma'], c['lambda_']))


def test_signature_and_namedtuples_match_the_reference():
    if not HAVE_REF:
        pytest.skip('reference archive not built')
    with reference() as ref:
        assert inspect.signature(b2.rl_utils.coma_error) == inspect.signature(ref.coma_error)
        assert b2.rl_utils.coma_data._fields == ref.coma_data._fields
        assert b2.rl_utils.coma_loss._fields == ref.coma_loss._fields
    assert b2.coma_error is b2.rl_utils.coma_error


@pytest.fixture
def dry(monkeypatch):
    rec = _RecordingLib()
    calls = []

    class _Counting:

        def __getattr__(self, name):
            fn = getattr(rec, name)

            def wrapped(*a):
                calls.append((name, a))
                return fn(*a)

            return wrapped

    monkeypatch.setattr(ops, 'lib', lambda: _Counting())
    monkeypatch.setattr(ops, 'require_cuda', lambda: None)
    monkeypatch.setattr(ops, 'compute_device', lambda *t: torch.device('cpu'))
    monkeypatch.setattr(ops, 'stream_ptr', lambda: 0)
    monkeypatch.setattr(ops, 'workspace', lambda dev: torch.zeros(1 << 18))
    monkeypatch.setattr(torch.cuda, 'device', lambda d: contextlib.nullcontext())
    yield calls


@pytest.mark.parametrize('name', ['smac_3s5z', 'w_bcast_a', 'n1'])
def test_marshalling_dry_run(dry, name):
    c = CASES[name]
    t = make_inputs(c)
    out = run(b2.rl_utils.coma_error, b2.rl_utils.coma_data, t, 'cpu', c, grads=('logit', 'q_value'))
    assert [n for n, _ in dry] == ['b200rl_coma_fwd', 'b200rl_coma_bwd']
    assert dry[0][1][6:10] == (c['T'], c['B'], c['A'], c['N'])
    assert out['grad_logit'].shape == out['grad_q_value'].shape == t['logit'].shape
    assert out['grad_target_q_value'] is None and out['grad_reward'] is None


def test_differentiable_returns_add_the_lambda_return_launches(dry):
    c = CASES['t2']
    run(b2.rl_utils.coma_error, b2.rl_utils.coma_data, make_inputs(c), 'cpu', c)
    names = [n for n, _ in dry]
    assert names[:2] == ['b200rl_lambda_returns', 'b200rl_coma_fwd']
    assert sorted(names[2:]) == sorted(['b200rl_coma_bwd', 'b200rl_scale', 'b200rl_lambda_returns_bwd'])
    assert dry[1][1][17] is not None  # dret: the forward launch writes d loss / d G


def test_no_gradient_wanted_writes_no_gradient(dry):
    c = CASES['t2']
    with torch.no_grad():
        loss = b2.rl_utils.coma_error(b2.rl_utils.coma_data(*(make_inputs(c)[k] for k in INPUTS)), 0.99, 0.95)
    assert all(l.grad_fn is None for l in loss)
    (name, args), = dry
    assert name == 'b200rl_coma_fwd' and args[12] is None and args[18] is None and args[19] is None


def _bad(t, **kw):
    t = dict(t)
    t.update(kw)
    return b2.rl_utils.coma_data(*(t[k] for k in INPUTS))


def _ref_raises(data):
    """the exception type the reference raises on ``data`` (None when it does not)"""
    with reference() as ref:
        try:
            ref.coma_error(data, 0.99, 0.95)
        except Exception as e:  # noqa: BLE001
            return type(e)
    return None


@pytest.mark.parametrize('shape', ['3d', '5d', 't1'])
def test_errors_match_the_reference(dry, shape):
    if not HAVE_REF:
        pytest.skip('reference archive not built')
    t = make_inputs(_case(20, 3, 2, 2, 4))
    if shape == '3d':
        data = _bad(t, logit=t['logit'][:, :, 0], action=t['action'][:, :, 0], q_value=t['q_value'][:, :, 0],
                    target_q_value=t['target_q_value'][:, :, 0])
    elif shape == '5d':
        data = _bad(t, logit=t['logit'][..., None, :], action=t['action'][..., None], q_value=t['q_value'][..., None, :],
                    target_q_value=t['target_q_value'][..., None, :])
    else:
        data = _bad(t, logit=t['logit'][:1], action=t['action'][:1], q_value=t['q_value'][:1],
                    target_q_value=t['target_q_value'][:1], reward=t['reward'][:1])
    exc = _ref_raises(data)
    assert exc is not None
    with pytest.raises(exc):
        b2.rl_utils.coma_error(data, 0.99, 0.95)
    assert dry == []


@pytest.mark.parametrize('dtype', [torch.float16, torch.bfloat16, torch.float64])
@pytest.mark.parametrize('field', ['logit', 'q_value', 'target_q_value', 'reward'])
def test_other_float_dtypes_raise_type_error(dry, dtype, field):
    t = make_inputs(CASES['t2'])
    with pytest.raises(TypeError):
        b2.rl_utils.coma_error(_bad(t, **{field: t[field].to(dtype)}), 0.99, 0.95)


def test_out_of_range_action_raises_index_error_when_checked(dry, monkeypatch):
    monkeypatch.setattr(ops, 'CHECK_INDICES', True)
    t = make_inputs(CASES['t2'])
    a = t['action'].clone()
    a[1, 2, 0] = t['logit'].shape[-1]
    with pytest.raises(IndexError):
        b2.rl_utils.coma_error(_bad(t, action=a), 0.99, 0.95)


def test_install_rebinds_coma_error_everywhere(monkeypatch):
    if not HAVE_REF:
        pytest.skip('reference archive not built')
    monkeypatch.setattr(ops, 'require_cuda', lambda: None)
    with reference() as ref:
        pkg = sys.modules['ding.rl_utils']
        orig = ref.coma_error
        monkeypatch.setattr(pkg, 'coma_error', orig, raising=False)
        policy = types.ModuleType('ding.policy.coma_install_test')
        policy.coma_error = orig  # `from ding.rl_utils import coma_data, coma_error` (policy/coma.py:7)
        sys.modules[policy.__name__] = policy
        try:
            done = b2.install()
            assert {m for m, n in done if n == 'coma_error'} == {'ding.rl_utils', 'ding.rl_utils.coma', policy.__name__}
            for mod in (pkg, ref, policy):
                assert mod.coma_error is b2.rl_utils.coma_error
        finally:
            b2.uninstall()
            del sys.modules[policy.__name__]
        for mod in (pkg, ref, policy):
            assert mod.coma_error is orig


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def _need_ref():
    if not HAVE_REF:
        pytest.skip('reference archive not built')


def _both(t, c, upstream=(1.0, 1.0, 1.0), grads=DIFF, device='cuda'):
    with reference() as ref:
        want = run(ref.coma_error, ref.coma_data, t, device, c, upstream, grads)
    got = run(b2.rl_utils.coma_error, b2.rl_utils.coma_data, t, device, c, upstream, grads)
    return want, got


@gpu
@pytest.mark.parametrize('upstream', sorted(UPSTREAMS))
@pytest.mark.parametrize('name', sorted(CASES))
def test_gpu_matches_the_reference(name, upstream):
    _need_ref()
    c = CASES[name]
    want, got = _both(make_inputs(c), c, UPSTREAMS[upstream])
    compare(want, got)


@gpu
@pytest.mark.parametrize('name', sorted(CASES))
def test_gpu_matches_the_fixtures(name):
    c, t, z = golden(name)
    compare_packed(z, run(b2.rl_utils.coma_error, b2.rl_utils.coma_data, t, 'cuda', c))


@gpu
@pytest.mark.parametrize('grads', [('logit', 'q_value'), ('logit', 'q_value', 'target_q_value'),
                                   ('logit', 'q_value', 'reward'), ('logit', ), ('q_value', ), ('target_q_value', )])
def test_gpu_requires_grad_combinations(grads):
    _need_ref()
    c = CASES['smac_mmm']
    t = make_inputs(c)
    want, got = _both(t, c, RECORD, grads)
    compare(want, got)
    x = {k: (v.cuda() if v is not None else None) for k, v in t.items()}
    for k in grads:
        x[k].requires_grad_(True)
    loss = b2.rl_utils.coma_error(b2.rl_utils.coma_data(*(x[k] for k in INPUTS)), 0.99, 0.8)
    if not ({'target_q_value', 'reward'} & set(grads)):
        fn = loss.policy_loss.grad_fn
        assert type(fn).__name__ == 'COMAFunctionBackward'
        assert [f is not None for f, _ in fn.next_functions][:2] == ['logit' in grads, 'q_value' in grads]


@gpu
def test_gpu_non_contiguous_operands():
    """every operand a non-contiguous view: a stride-2 slice of the last dim of (T, B, A, N) storage, transposed (T, B) /
    (T, B, A) storage; the gradients reach the storage through the views"""
    _need_ref()
    c = _case(31, 8, 5, 3, 7, 'rand', mask='inf')
    t = make_inputs(c)

    def storage(v):
        if v.dim() == 4:
            s = torch.zeros(*v.shape[:-1], 2 * v.shape[-1], dtype=v.dtype)
            s[..., ::2] = v
            return s.cuda()
        return v.transpose(0, 1).contiguous().cuda()

    def view(k, s):
        return s[..., ::2] if s.dim() == 4 else s.transpose(0, 1)

    res = []
    for fn, cls in ((None, None), (b2.rl_utils.coma_error, b2.rl_utils.coma_data)):
        with reference() as ref:
            f, k_ = (ref.coma_error, ref.coma_data) if fn is None else (fn, cls)
            st = {k: storage(v) for k, v in t.items()}
            for k in DIFF:
                st[k].requires_grad_(True)
            xs = {k: view(k, s) for k, s in st.items()}
            for k in INPUTS:
                assert not xs[k].is_contiguous() and torch.equal(xs[k].detach().cpu(), t[k]), k
            loss = f(k_(*(xs[k] for k in INPUTS)), c['gamma'], c['lambda_'])
            sum(u * l for u, l in zip(RECORD, loss)).backward()
            out = {k: getattr(loss, k).detach().double().cpu().numpy() for k in ('policy_loss', 'q_value_loss',
                                                                                 'entropy_loss')}
            out.update({'grad_' + k: st[k].grad.double().cpu().numpy() for k in DIFF})
            res.append(out)
    compare(*res)


@gpu
def test_gpu_repeated_and_interleaved_backward():
    _need_ref()
    c = CASES['smac_3s5z']
    t = make_inputs(c)
    outs = []
    for fn, cls in ((None, None), (b2.rl_utils.coma_error, b2.rl_utils.coma_data)):
        with reference() as ref:
            f, k = (ref.coma_error, ref.coma_data) if fn is None else (fn, cls)
            x = {n: (v.cuda() if v is not None else None) for n, v in t.items()}
            for n in ('logit', 'q_value'):
                x[n].requires_grad_(True)
            l1 = f(k(*(x[n] for n in INPUTS)), 0.99, 0.8)
            l2 = f(k(*(x[n] for n in INPUTS)), 0.99, 0.8)
            sum(u * l for u, l in zip(RECORD, l1)).backward(retain_graph=True)
            sum(u * l for u, l in zip((1.0, 1.0, 1.0), l2)).backward(retain_graph=True)
            sum(u * l for u, l in zip(RECORD, l1)).backward(retain_graph=True)
            sum(u * l for u, l in zip((0.37, 0.0, 2.0), l1)).backward()
            outs.append({'grad_' + n: x[n].grad.double().cpu().numpy() for n in ('logit', 'q_value')})
    compare(outs[0], outs[1])


@gpu
def test_gpu_record_match_returns_without_writing():
    c = CASES['smac_3s5z']
    x = {k: (v.cuda() if v is not None else None) for k, v in make_inputs(c).items()}
    for n in ('logit', 'q_value'):
        x[n].requires_grad_(True)
    ops.ppo_hint(x['logit'].device, 'coma').copy_(torch.tensor([0.001, 1.0, -0.01, 0.0]))
    loss = b2.rl_utils.coma_error(b2.rl_utils.coma_data(*(x[n] for n in INPUTS)), 0.99, 0.8)
    ctx = loss.policy_loss.grad_fn
    written = ctx.spec[0].data_ptr()  # no reference kept: autograd adopts a gradient only while nothing else holds it
    sentinel = ctx.spec[0].clone()
    (0.001 * loss.policy_loss + 1 * loss.q_value_loss - 0.01 * loss.entropy_loss).backward()
    assert x['logit'].grad.data_ptr() == written  # adopted without a copy
    assert torch.equal(x['logit'].grad, sentinel)


@gpu
@pytest.mark.parametrize('name', ['smac_2c64zg', 'n257', 'ref_weight'])
def test_gpu_deterministic(name):
    c = CASES[name]
    t = make_inputs(c)
    a = run(b2.rl_utils.coma_error, b2.rl_utils.coma_data, t, 'cuda', c, RECORD)
    b = run(b2.rl_utils.coma_error, b2.rl_utils.coma_data, t, 'cuda', c, RECORD)
    for k in a:
        if a[k] is not None:
            assert np.array_equal(a[k], b[k], equal_nan=True), k


@gpu
@pytest.mark.parametrize('name', ['smac_3s5z', 'w_bcast_a', 'n257'])
def test_gpu_fullgraph_compile_is_bit_identical_to_eager(name):
    c = CASES[name]
    t = make_inputs(c)

    def step(logit, action, q_value, target_q_value, reward, weight):
        loss = b2.rl_utils.coma_error(b2.rl_utils.coma_data(logit, action, q_value, target_q_value, reward, weight),
                                      c['gamma'], c['lambda_'])
        return loss.policy_loss, loss.q_value_loss, loss.entropy_loss

    torch._dynamo.reset()
    compiled = torch.compile(step, fullgraph=True, backend='inductor')
    res = []
    for fn in (step, compiled):
        x = {k: (v.cuda() if v is not None else None) for k, v in t.items()}
        for n in ('logit', 'q_value'):
            x[n].requires_grad_(True)
        out = fn(*(x[n] for n in INPUTS))
        sum(u * l for u, l in zip(RECORD, out)).backward()
        res.append([o.detach().cpu() for o in out] + [x['logit'].grad.cpu(), x['q_value'].grad.cpu()])
    for a, b in zip(*res):
        assert torch.equal(a, b) or (torch.isnan(a).all() and torch.isnan(b).all())


def ported_inputs():
    """the inputs of ding/rl_utils/tests/test_coma.py, drawn in its order from torch's seeded global generator:
    {'none' | 'random': (logit, action, reward, q_value, target_q_value, weight)}"""
    state = torch.random.get_rng_state()
    try:
        torch.manual_seed(0)
        T, B, A, N = 128, 4, 8, 32
        random_weight = torch.rand(T, B, A) + 1
        out = {}
        for name, weight in (('none', None), ('random', random_weight)):
            logit = torch.randn(T, B, A, N)
            action = torch.randint(0, N, size=(T, B, A))
            reward = torch.rand(T, B)
            q_value = torch.randn(T, B, A, N)
            target_q_value = torch.randn(T, B, A, N)
            out[name] = (logit, action, reward, q_value, target_q_value, weight)
        return out
    finally:
        torch.random.set_rng_state(state)


def ported_test(coma_data, coma_error, inputs, device):
    """the body of ding/rl_utils/tests/test_coma.py on ``device``; -> the losses and gradients"""
    logit, action, reward, q_value, target_q_value, weight = (x.to(device) if x is not None else None for x in inputs)
    logit.requires_grad_(True)
    q_value.requires_grad_(True)
    target_q_value.requires_grad_(True)
    data = coma_data(logit, action, q_value, target_q_value, reward, weight)
    loss = coma_error(data, 0.99, 0.95)
    assert all([l.shape == tuple() for l in loss])
    assert logit.grad is None
    assert q_value.grad is None
    total_loss = sum(loss)
    total_loss.backward()
    assert isinstance(logit.grad, torch.Tensor)
    assert isinstance(q_value.grad, torch.Tensor)
    return {'losses': torch.stack(list(loss)).detach().double().cpu().numpy(),
            **{'grad_' + k: v.grad.double().cpu().numpy() for k, v in (('logit', logit), ('q_value', q_value),
                                                                        ('target_q_value', target_q_value))}}


@gpu
@pytest.mark.parametrize('weight', ['none', 'random'])
def test_gpu_ported_reference_test(weight):
    """ding/rl_utils/tests/test_coma.py on the library, against the reference's values stored in the fixture"""
    z = np.load(os.path.join(GOLDEN_DIR, 'ported_reference_test.npz'))
    compare_packed(z, ported_test(b2.rl_utils.coma_data, b2.rl_utils.coma_error, ported_inputs()[weight], 'cuda'),
                   weight + '_')


class _StandIn(torch.nn.Module):
    """a stand-in for COMA's actor / critic: linear heads on a shared observation"""

    def __init__(self, obs, A, N):
        super().__init__()
        self.actor = torch.nn.Linear(obs, N)
        self.critic = torch.nn.Linear(obs + A, N)


def _policy_block(model, target, batch, coma_data, coma_error):
    """COMAPolicy._forward_learn's loss block (policy/coma.py:205-218) on the stand-in"""
    obs, onehot = batch['obs'], batch['agent_onehot']
    q_value = model.critic(torch.cat([obs, onehot], -1))
    with torch.no_grad():
        target_q_value = target.critic(torch.cat([obs, onehot], -1))
    logit = model.actor(obs)
    logit[batch['action_mask'] == 0.0] = -9999999
    data = coma_data(logit, batch['action'], q_value, target_q_value, batch['reward'], batch['weight'])
    coma_loss = coma_error(data, 0.99, 0.8)
    total_loss = 0.001 * coma_loss.policy_loss + 1 * coma_loss.q_value_loss - 0.01 * coma_loss.entropy_loss
    model.zero_grad()
    total_loss.backward()
    return [p.grad.double().cpu().numpy() for p in model.parameters()], total_loss.item()


@gpu
def test_gpu_coma_policy_loss_block_before_and_after_install():
    _need_ref()
    T, B, A, N, obs = 10, 32, 8, 14, 24
    g = torch.Generator().manual_seed(40)
    model, target = _StandIn(obs, A, N).cuda(), _StandIn(obs, A, N).cuda()
    mask = (torch.rand(T, B, A, N, generator=g) < 0.7).float()
    action = torch.randint(0, N, (T, B, A), generator=g)
    mask.scatter_(-1, action.unsqueeze(-1), 1.0)
    batch = {'obs': torch.randn(T, B, A, obs, generator=g), 'agent_onehot': torch.eye(A).expand(T, B, A, A).contiguous(),
             'action_mask': mask, 'action': action, 'reward': torch.rand(T, B, generator=g), 'weight': None}
    batch = {k: (v.cuda() if v is not None else None) for k, v in batch.items()}
    with reference() as ref:
        policy = types.ModuleType('ding.policy.coma_block_test')
        policy.coma_data, policy.coma_error = ref.coma_data, ref.coma_error
        sys.modules[policy.__name__] = policy
        try:
            want, want_total = _policy_block(model, target, batch, policy.coma_data, policy.coma_error)
            b2.install()
            try:
                assert policy.coma_error is b2.rl_utils.coma_error
                for _ in range(2):  # the second step verifies the record the first one left
                    got, got_total = _policy_block(model, target, batch, policy.coma_data, policy.coma_error)
                    assert abs(got_total - want_total) <= 1e-5 + 1e-5 * abs(want_total)
                    for i, (w_, g_) in enumerate(zip(want, got)):
                        close(w_, g_, 'param %d' % i)
            finally:
                b2.uninstall()
        finally:
            del sys.modules[policy.__name__]
