"""FQF's fraction loss, ``fqf_calculate_fraction_loss`` (ding/rl_utils/td.py:1466-1513), on the fqf_fraction kernels of
csrc/quantile.cu.

CPU (``-m "not gpu"``):
  * the fixtures in ``tests/golden/fqf_fraction/`` hold the seeded inputs, and the live reference reproduces their outputs;
  * the float64 restatement (tests/fqf_fraction_oracle.py) agrees with the fixtures and with the live reference;
  * every call marshals against the ctypes prototypes (recording stand-in of test_reference_suite.py), with the views'
    own pointers and strides (no copy), one forward and one backward launch;
  * the reference's AssertionErrors, and TypeError for dtypes other than fp32.
GPU: the loss within 1e-5 + 1e-5 * |ref| and d loss / d quantiles bit-exact against the reference run on the same CUDA
tensors, for upstream gradients 1, 0.37 and 0; against the fixtures (minted on the CPU, where torch divides by B instead of
multiplying by fp32(1 / B): within 3e-7 relative for u = 0.37) and the restatement; and FQFPolicy's loss block
(policy/fqf.py:239-248) with the reference functions and after ``install()``.
"""
import contextlib
import glob
import json
import os

import numpy as np
import pytest
import torch

import di_engine_b200 as b2
from di_engine_b200 import ops
from oracle import ref_loader
from tests import fqf_fraction_oracle as oracle
from tests.test_reference_suite import _RecordingLib

HAVE_REF = ref_loader.available()
GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'fqf_fraction')
INPUTS = ('q_tau_i', 'q_value', 'quantiles', 'actions')
UPSTREAM = (1.0, 0.37)


def _case(seed, B, N, A, rows=None):
    """rows: 'ties' (values on an integer grid, so s_i ties its neighbours and h; one all-equal row, one increasing and one
    decreasing row), 'inf' (+inf, -inf and NaN in q_value)"""
    return dict(seed=seed, B=B, N=N, A=A, rows=rows)


CASES = {
    'pong': _case(1, 32, 32, 6),
    'cartpole': _case(2, 64, 32, 2),
    'b1_n2_a1': _case(3, 1, 2, 1),
    'n33_a64': _case(4, 3, 33, 64),
    'n200': _case(5, 5, 200, 3),
    'ties': _case(6, 32, 32, 6, 'ties'),
    'inf_nan': _case(7, 12, 8, 4, 'inf'),
}


def make_inputs(c, device='cpu'):
    """seeded inputs; ``quantiles`` is a zero-padded cumsum of a softmax, as FQF's head builds it (model/common/head.py:744-760)"""
    g = torch.Generator(device=device).manual_seed(c['seed'])
    B, N, A = c['B'], c['N'], c['A']

    def randn(*s):
        return torch.randn(*s, generator=g, device=device)

    if c['rows'] == 'ties':
        q_value = torch.randint(-2, 3, (B, N, A), generator=g, device=device).float()
        q_tau_i = torch.randint(-2, 3, (B, N - 1, A), generator=g, device=device).float()
        q_value[0], q_tau_i[0] = 1.0, 1.0  # all equal
        up = torch.arange(2 * N - 1, device=device).float()  # h_0 < s_0 < h_1 < s_1 < ... < h_{N-1}
        q_value[1], q_tau_i[1] = up[0::2, None], up[1::2, None]
        q_value[2], q_tau_i[2] = -up[0::2, None], -up[1::2, None]
    else:
        q_value, q_tau_i = randn(B, N, A), randn(B, N - 1, A)
    actions = torch.randint(0, A, (B, ), generator=g, device=device)
    actions[0], actions[-1] = 0, A - 1
    if c['rows'] == 'inf':
        for b, v in ((0, float('inf')), (1, float('-inf')), (2, float('nan'))):
            q_value[b, 1, actions[b]] = v
        q_value[3, 0, actions[3]] = float('inf')  # h_0: the left neighbour of s_0
        q_value[4, N - 1, actions[4]] = float('nan')  # h_{N-1}: the right neighbour of s_{N-2}
    p = torch.softmax(randn(B, N), 1)
    quantiles = torch.cat([torch.zeros(B, 1, device=device), torch.cumsum(p, 1)], 1)
    return {'q_tau_i': q_tau_i, 'q_value': q_value, 'quantiles': quantiles, 'actions': actions}


def run(api, t, dev, upstream=1.0):
    """-> {'loss', 'grad'}: the loss and d (upstream * loss) / d quantiles, float64 numpy"""
    q_value = t['q_value'].detach().clone().to(dev).requires_grad_(True)
    quantiles = t['quantiles'].detach().clone().to(dev).requires_grad_(True)
    loss = api.fqf_calculate_fraction_loss(t['q_tau_i'].to(dev), q_value, quantiles, t['actions'].to(dev))
    loss.backward(torch.tensor(upstream, device=loss.device))
    assert q_value.grad is None
    return {'loss': loss.detach().cpu().double().numpy(), 'grad': quantiles.grad.cpu().double().numpy()}


def close_loss(got, want):
    assert np.allclose(got, want, rtol=1e-5, atol=1e-5, equal_nan=True), (float(got), float(want))


def same_bits(got, want):
    assert np.array_equal(np.asarray(got, np.float32), np.asarray(want, np.float32), equal_nan=True), \
        float(np.nanmax(np.abs(np.asarray(got) - np.asarray(want))))


def close_grad(got, want, tol=1e-5):
    fin = want[np.isfinite(want)]
    scale = max(1.0, float(np.max(np.abs(fin)))) if fin.size else 1.0
    assert np.allclose(got, want, rtol=tol, atol=tol * scale, equal_nan=True), float(np.nanmax(np.abs(got - want)))


def load_fixture(name):
    with np.load(os.path.join(GOLDEN_DIR, name + '.npz'), allow_pickle=False) as z:
        d = {k: z[k] for k in z.files}
    case = json.loads(str(d.pop('case')))
    return case, {k: torch.from_numpy(d['in_' + k]) for k in INPUTS}, d


# =================================================================================================================
# CPU
# =================================================================================================================
def test_fixture_set_matches_cases():
    assert sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN_DIR, '*.npz'))) == sorted(CASES)


@pytest.mark.parametrize('name', sorted(CASES))
def test_fixture_inputs_are_the_seeded_case(name):
    case, t, _ = load_fixture(name)
    assert case == CASES[name]
    want = make_inputs(case)
    for k in INPUTS:
        assert t[k].dtype == want[k].dtype and np.array_equal(t[k].numpy(), want[k].numpy(), equal_nan=True), k


def test_fixtures_cover_the_edges():
    _, t, d = load_fixture('ties')
    s = t['q_tau_i'].gather(2, t['actions'][:, None, None].expand(-1, 31, 1))[..., 0]
    h = t['q_value'].gather(2, t['actions'][:, None, None].expand(-1, 32, 1))[..., 0]
    assert (s[:, 1:] == s[:, :-1]).any() and (s == h[:, :-1]).any() and (s == h[:, 1:]).any()
    _, _, d = load_fixture('inf_nan')
    assert np.isnan(d['out_loss']) and np.isnan(d['out_grad_u1']).any() and np.isinf(d['out_grad_u1']).any()


@pytest.mark.skipif(not HAVE_REF, reason='reference not importable here')
@pytest.mark.parametrize('name', sorted(CASES))
def test_fixture_outputs_are_the_live_reference(name):
    _, t, d = load_fixture(name)
    ref = ref_loader.load()
    for u in UPSTREAM:
        got = run(ref, t, 'cpu', u)
        same_bits(got['loss'], d['out_loss'])
        same_bits(got['grad'], d[grad_key(u)])


def grad_key(u):
    return 'out_grad_u' + ('1' if u == 1.0 else str(u).replace('.', ''))


@pytest.mark.parametrize('name', sorted(CASES))
def test_restatement_matches_the_fixtures(name):
    _, t, d = load_fixture(name)
    for u in UPSTREAM:
        loss, grad = oracle.fraction_loss(t['q_tau_i'], t['q_value'], t['quantiles'], t['actions'], u)
        close_loss(loss, d['out_loss'])
        close_grad(grad, d[grad_key(u)])


@pytest.mark.skipif(not HAVE_REF, reason='reference not importable here')
@pytest.mark.parametrize('B,N,A', [(3, 2, 1), (64, 32, 6), (200, 200, 2), (1025, 33, 64)])
def test_restatement_matches_the_live_reference(B, N, A):
    t = make_inputs(_case(11 + N, B, N, A))
    got = run(ref_loader.load(), t, 'cpu', 0.37)
    loss, grad = oracle.fraction_loss(t['q_tau_i'], t['q_value'], t['quantiles'], t['actions'], 0.37)
    close_loss(loss, got['loss'])
    close_grad(grad, got['grad'])


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


@pytest.mark.filterwarnings('ignore:invalid value encountered in cast')  # the stand-in leaves outputs uninitialised
@pytest.mark.parametrize('name', sorted(CASES))
def test_marshalling_dry_run(dry, name):
    case = CASES[name]
    t = make_inputs(case)
    B, N = case['B'], case['N']
    res = run(b2.rl_utils, t, 'cpu')
    assert [c[0] for c in dry] == ['b200rl_fqf_fraction_fwd', 'b200rl_fqf_fraction_bwd']
    assert res['loss'].shape == () and res['grad'].shape == (B, N + 1)
    fwd = dry[0][1]
    assert fwd[4:8] == (B, N, case['A'], case['A'])


def test_views_reach_the_kernel_without_a_copy(dry):
    B, N, A = 8, 5, 3
    t = make_inputs(_case(9, B, N, A))
    qt = t['q_tau_i'].permute(0, 2, 1).contiguous().permute(0, 2, 1)  # (B, N-1, A) with the action axis outermost
    qv_base = torch.randn(B, N + 2, A + 1)
    qv = qv_base[:, 1:N + 1, :A].requires_grad_(True)
    qn_base = t['quantiles'].t().contiguous().requires_grad_(True)
    qn = qn_base.t()  # (B, N+1), column-major
    loss = b2.fqf_calculate_fraction_loss(qt, qv, qn, t['actions'])
    name, a = dry[0]
    assert a[:3] == (qt.data_ptr(), qv.data_ptr(), qn.data_ptr())
    assert a[8:16] == qt.stride() + qv.stride() + qn.stride()
    loss.backward()
    assert qn_base.grad.shape == (N + 1, B) and qv.grad is None


def test_no_grad_fn_without_quantiles_grad(dry):
    t = make_inputs(CASES['pong'])
    for api in _apis():
        loss = api.fqf_calculate_fraction_loss(t['q_tau_i'], t['q_value'].requires_grad_(True), t['quantiles'],
                                               t['actions'])
        assert loss.grad_fn is None and not loss.requires_grad


def _apis():
    return [b2.rl_utils] + ([ref_loader.load()] if HAVE_REF else [])


def test_assertions_match_the_reference(dry):
    t = make_inputs(CASES['pong'])
    qt, qv, qn, act = t['q_tau_i'], t['q_value'], t['quantiles'], t['actions']
    for api in _apis():
        f = api.fqf_calculate_fraction_loss
        with pytest.raises(AssertionError):  # td.py:1480
            f(qt, qv, qn.requires_grad_(True), act)
        qv_g = qv.clone().requires_grad_(True)
        with pytest.raises(AssertionError):  # td.py:1487: N quantiles instead of N-1
            f(qv, qv_g, qn, act)
        with pytest.raises(AssertionError):  # td.py:1507: quantiles (B, N)
            f(qt, qv_g, qn[:, :-1], act)
        with pytest.raises(AssertionError):  # td.py:1453: batch of actions
            f(qt, qv_g, qn, act[:-1])


@pytest.mark.parametrize('dtype', [torch.float64, torch.float16, torch.bfloat16])
@pytest.mark.parametrize('which', ['q_tau_i', 'q_value', 'quantiles'])
def test_other_float_dtypes_raise_type_error(dry, which, dtype):
    t = make_inputs(CASES['pong'])
    t[which] = t[which].to(dtype)
    with pytest.raises(TypeError, match=which):
        b2.fqf_calculate_fraction_loss(t['q_tau_i'], t['q_value'].requires_grad_(True), t['quantiles'], t['actions'])


def test_out_of_range_action_raises_with_index_checks(dry, monkeypatch):
    monkeypatch.setattr(ops, 'CHECK_INDICES', True)
    t = make_inputs(CASES['pong'])
    t['actions'][3] = 6
    with pytest.raises(IndexError, match='out of range for 6 classes'):
        b2.fqf_calculate_fraction_loss(t['q_tau_i'], t['q_value'].requires_grad_(True), t['quantiles'], t['actions'])


# =================================================================================================================
# GPU
# =================================================================================================================
def reference_or_skip():
    if not HAVE_REF:
        pytest.skip('reference not importable here')
    return ref_loader.load()


def check_against_reference(t, ref, upstreams=(0.0, 1.0, 0.37)):
    """bit-exact gradient and the loss at 1e-5 against the reference on the same CUDA tensors, and against the restatement
    (for the last upstream gradient)"""
    for u in upstreams:
        got, want = run(b2.rl_utils, t, 'cuda', u), run(ref, t, 'cuda', u)
        close_loss(got['loss'], want['loss'])
        same_bits(got['grad'], want['grad'])
    loss, grad = oracle.fraction_loss(*(t[k].cpu() for k in INPUTS), upstreams[-1])
    close_loss(got['loss'], loss)
    close_grad(got['grad'], grad)


@pytest.mark.gpu
@pytest.mark.parametrize('name', sorted(CASES))
def test_fixture_cases(name):
    _, t, d = load_fixture(name)
    got = run(b2.rl_utils, t, 'cuda', 1.0)
    close_loss(got['loss'], d['out_loss'])
    same_bits(got['grad'], d['out_grad_u1'])  # fp32(1 / B) is what both the division and the reciprocal give
    got = run(b2.rl_utils, t, 'cuda', 0.37)
    assert np.allclose(got['grad'], d['out_grad_u037'], rtol=3e-7, atol=0, equal_nan=True)
    if HAVE_REF:
        check_against_reference(t, ref_loader.load())


SIZES_B = [1, 32, 64, 1024, 1025, 65536]
SIZES_N = [2, 32, 33, 200]
ACTIONS = [1, 2, 6, 64]


@pytest.mark.gpu
@pytest.mark.parametrize('N', SIZES_N)
@pytest.mark.parametrize('B', SIZES_B)
def test_shapes_against_reference(B, N):
    ref = reference_or_skip()
    A = ACTIONS[(SIZES_B.index(B) + SIZES_N.index(N)) % 4]
    if B * N * A > 1 << 24:
        A = 6
    check_against_reference(make_inputs(_case(100 + B % 97 + N, B, N, A), 'cuda'), ref)


@pytest.mark.gpu
@pytest.mark.parametrize('A', ACTIONS)
def test_action_counts_against_reference(A):
    check_against_reference(make_inputs(_case(200 + A, 257, 32, A), 'cuda'), reference_or_skip())


@pytest.mark.gpu
@pytest.mark.parametrize('rows', ['ties', 'inf'])
@pytest.mark.parametrize('B', [64, 1025])
def test_edge_rows_against_reference(rows, B):
    check_against_reference(make_inputs(_case(300 + B, B, 33, 6, rows), 'cuda'), reference_or_skip())


@pytest.mark.gpu
@pytest.mark.parametrize('B', [32, 1025])
def test_strided_views_against_reference(B):
    """transposed / sliced q_tau_i, q_value and quantiles: the gradient lands in the leaf behind the view"""
    ref = reference_or_skip()
    N, A = 32, 6
    t = make_inputs(_case(400 + B, B, N, A), 'cuda')
    outs = []
    for api in (b2.rl_utils, ref):
        qt = t['q_tau_i'].permute(0, 2, 1).contiguous().permute(0, 2, 1)
        qv = torch.cat([t['q_value'], t['q_value']], 2)[:, :, ::2]
        leaf = t['quantiles'].t().contiguous().requires_grad_(True)
        loss = api.fqf_calculate_fraction_loss(qt, qv.requires_grad_(True), leaf.t(), t['actions'])
        loss.backward(torch.tensor(0.37, device='cuda'))
        outs.append((loss.item(), leaf.grad.cpu().numpy()))
    close_loss(outs[0][0], outs[1][0])
    same_bits(outs[0][1], outs[1][1])


@pytest.mark.gpu
def test_quantiles_without_grad_on_device():
    ref = reference_or_skip()
    t = make_inputs(CASES['pong'], 'cuda')
    losses = []
    for api in (b2.rl_utils, ref):
        loss = api.fqf_calculate_fraction_loss(t['q_tau_i'], t['q_value'].clone().requires_grad_(True), t['quantiles'],
                                               t['actions'])
        assert loss.grad_fn is None and loss.is_cuda
        losses.append(loss.item())
    close_loss(*losses)


@pytest.mark.gpu
def test_backward_sequences_against_reference():
    """repeated backward with retain_graph (the second recomputes), a scaled one, and a backward after a second forward"""
    ref = reference_or_skip()
    t1 = make_inputs(_case(500, 64, 32, 6), 'cuda')
    t2 = make_inputs(_case(501, 64, 32, 6), 'cuda')
    grads = []
    for api in (b2.rl_utils, ref):
        q1 = t1['quantiles'].clone().requires_grad_(True)
        q2 = t2['quantiles'].clone().requires_grad_(True)
        l1 = api.fqf_calculate_fraction_loss(t1['q_tau_i'], t1['q_value'].clone().requires_grad_(True), q1, t1['actions'])
        l1.backward(retain_graph=True)
        g1 = q1.grad.clone()
        l1.backward(retain_graph=True)
        g2 = q1.grad.clone()
        l2 = api.fqf_calculate_fraction_loss(t2['q_tau_i'], t2['q_value'].clone().requires_grad_(True), q2, t2['actions'])
        l1.backward(torch.tensor(0.37, device='cuda'))
        g3 = q1.grad.clone()
        (3.0 * l2).backward()
        grads.append([g.cpu().numpy() for g in (g1, g2, g3, q2.grad)])
    for a, b in zip(*grads):
        same_bits(a, b)


@pytest.mark.gpu
def test_host_buffers():
    _, t, d = load_fixture('pong')
    got = run(b2.rl_utils, t, 'cpu', 1.0)
    close_loss(got['loss'], d['out_loss'])
    same_bits(got['grad'], d['out_grad_u1'])


@pytest.mark.gpu
def test_out_of_range_action_gives_nan():
    t = make_inputs(CASES['pong'], 'cuda')
    t['actions'][5] = 6
    got = run(b2.rl_utils, t, 'cuda', 1.0)
    assert np.isnan(got['loss'])
    assert np.isnan(got['grad'][5, 1:-1]).all() and not np.isnan(np.delete(got['grad'], 5, 0)).any()
    assert (got['grad'][:, [0, -1]] == 0).all()


# ---- FQFPolicy's loss block (policy/fqf.py:239-248) on a stand-in model -------------------------------------------------
def fqf_block(rl, model, data, gamma=0.99, nstep=1, kappa=1.0, ent_coef=0.01):
    ret = model()
    q_value, quantiles, quantiles_hats, q_tau_i, entropies = (ret[k] for k in
                                                              ('q', 'quantiles', 'quantiles_hats', 'q_tau_i', 'entropies'))
    data_n = rl.fqf_nstep_td_data(q_value, data['target_q'], data['action'], data['target_action'], data['reward'],
                                  data['done'], quantiles_hats, data['weight'])
    entropy_loss = -ent_coef * entropies.mean()
    fraction_loss = rl.fqf_calculate_fraction_loss(q_tau_i.detach(), q_value, quantiles, data['action']) + entropy_loss
    quantile_loss, td_error_per_sample = rl.fqf_nstep_td_error(data_n, gamma, nstep=nstep, kappa=kappa)
    fraction_loss.backward(retain_graph=True)
    quantile_loss.backward()
    return fraction_loss.item(), quantile_loss.item()


class StandIn(torch.nn.Module):
    """the fraction-proposal part of FQF's head (model/common/head.py:744-760) over learnable tensors"""

    def __init__(self, B, N, A, g):
        super().__init__()
        self.frac = torch.nn.Parameter(torch.randn(B, N, generator=g))
        self.q = torch.nn.Parameter(torch.randn(B, N, A, generator=g))
        self.tau = torch.nn.Parameter(torch.randn(B, N - 1, A, generator=g))

    def forward(self):
        log_q = torch.log_softmax(self.frac, 1)
        q = log_q.exp()
        entropies = -(log_q * q).sum(-1, keepdim=True)
        quantiles = torch.cat([torch.zeros_like(q[:, :1]), torch.cumsum(q, 1)], 1)
        hats = (quantiles[:, 1:] + quantiles[:, :-1]).detach() / 2.
        return {'q': self.q * (1.0 + hats[:, :, None]), 'quantiles': quantiles, 'quantiles_hats': hats,
                'q_tau_i': self.tau + quantiles[:, 1:-1, None], 'entropies': entropies}


@pytest.mark.gpu
@pytest.mark.parametrize('B,N,A', [(32, 32, 6), (64, 32, 2)])
def test_fqf_policy_loss_block_before_and_after_install(B, N, A):
    ref = reference_or_skip()
    g = torch.Generator().manual_seed(600 + B)
    model = StandIn(B, N, A, g).cuda()
    data = {'target_q': torch.randn(B, N, A, generator=g).cuda(), 'action': torch.randint(0, A, (B, ), generator=g).cuda(),
            'target_action': torch.randint(0, A, (B, ), generator=g).cuda(), 'reward': torch.randn(1, B, generator=g).cuda(),
            'done': torch.randint(0, 2, (B, ), generator=g).float().cuda(), 'weight': None}
    fns = ('fqf_calculate_fraction_loss', 'fqf_nstep_td_error')
    runs = []
    for installed in (False, True):
        model.zero_grad(set_to_none=True)
        try:
            if installed:
                b2.install()
                assert all(getattr(ref, n) is getattr(b2.rl_utils, n) for n in fns)
            losses = fqf_block(ref, model, data)
        finally:
            b2.uninstall()
        runs.append((losses, {k: p.grad.cpu().numpy() for k, p in model.named_parameters() if p.grad is not None}))
    assert not any(getattr(ref, n) is getattr(b2.rl_utils, n) for n in fns)
    (want_l, want_g), (got_l, got_g) = runs
    for a, b in zip(got_l, want_l):
        close_loss(a, b)
    assert set(got_g) == set(want_g) == {'frac', 'q'}
    close_grad(got_g['frac'], want_g['frac'])
    close_grad(got_g['q'], want_g['q'])
