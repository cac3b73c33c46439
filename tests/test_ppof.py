"""PPOFPolicy's advantage recompute (``ppof_gae_returns``: ding/policy/ppof.py:160-210 in one call) and ``symlog`` /
``inv_symlog`` (ding/rl_utils/value_rescale.py:37-66), on the kernels of csrc/policy.cu.

CPU (``-m "not gpu"``):
  * the fixtures in ``tests/golden/ppof/`` hold the seeded inputs, and the restatement of ppof.py (tests/ppof_oracle.py)
    around the live reference reproduces their outputs bit for bit;
  * every call marshals against the ctypes prototypes: ONE ``b200rl_gae_returns_norm`` call for every mode and shape, with
    the mode's code, std, mu / sigma and a decode scratch exactly where the multi-launch path needs one;
  * bad arguments raise before any call, and the built library rejects them before any launch (B200RL_ERR_ARG);
  * ``install()`` rebinds ``symlog`` / ``inv_symlog`` in a module holding PPOF's imported names, ``uninstall()`` restores them.
GPU: the semantics table of every mode against the restatement on the CPU and on the same CUDA tensors, at n = 1 ... 30000
and (T, B) = (33, 36), (128, 4096); the fixtures; the kernels each path launches; ``symlog`` / ``inv_symlog`` forward and
backward against the reference on the same CUDA tensors.
"""
import contextlib
import glob
import json
import os
import sys
import types

import numpy as np
import pytest
import torch

import di_engine_b200 as b2
from di_engine_b200 import _lib, ops
from oracle import ref_loader
from tests import ppof_oracle
from tests.test_reference_suite import _RecordingLib

HAVE_REF = ref_loader.available()
GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'ppof')
MODES = ('baseline', 'value_rescale', 'symlog', 'popart')
GAMMA, LAMBDA = 0.99, 0.95
INPUTS = ('pred', 'next_pred', 'reward', 'done', 'traj_flag', 'mu', 'sigma')


def _case(seed, mode, shape, done='float', traj=True, special=None, col=False):
    """shape: (n,) or (T, B); done: 'float' | 'bool' | 'none' (traj_flag None too); traj: traj_flag = done plus segment
    cuts; special 'inf_nan': preds whose inv_symlog overflows fp32 (|x| >= 89) and NaNs; col: value (n, 1) against an (n,)
    reward (PopArt's prediction, gae.py:56-59)"""
    return dict(seed=seed, mode=mode, shape=list(shape), done=done, traj=traj, special=special, col=col)


CASES = {
    'baseline_n128': _case(1, 'baseline', (128, )),
    'baseline_n400_bool': _case(2, 'baseline', (400, ), done='bool'),
    'baseline_n400_none': _case(3, 'baseline', (400, ), done='none', traj=False),
    'baseline_n400_inf_nan': _case(4, 'baseline', (400, ), special='inf_nan'),
    'value_rescale_n128': _case(5, 'value_rescale', (128, )),
    'value_rescale_n400_bool': _case(6, 'value_rescale', (400, ), done='bool'),
    'value_rescale_n400_none': _case(7, 'value_rescale', (400, ), done='none', traj=False),
    'symlog_n128': _case(8, 'symlog', (128, )),
    'symlog_n400_none': _case(9, 'symlog', (400, ), done='none', traj=False),
    'symlog_n400_inf_nan': _case(10, 'symlog', (400, ), special='inf_nan'),
    'popart_n128_col': _case(11, 'popart', (128, ), col=True),
    'popart_n400_col_bool': _case(12, 'popart', (400, ), done='bool', col=True),
    'popart_n400_none': _case(13, 'popart', (400, ), done='none', traj=False),
}
STD = 1.7320508  # a RunningMeanStd.std


def make_inputs(c, device='cpu'):
    g = torch.Generator().manual_seed(c['seed'])
    shape = tuple(c['shape'])
    scale = 3.0 if c['mode'] in ('symlog', 'value_rescale') else 1.0
    pred = torch.randn(*shape, generator=g) * scale
    next_pred = torch.randn(*shape, generator=g) * scale
    reward = torch.randn(*shape, generator=g)
    done = torch.rand(*shape, generator=g) < 0.03
    if c['special'] == 'inf_nan':
        n = pred.numel()
        idx = torch.randperm(n, generator=g)[:12]
        vals = torch.tensor([89.0, -89.5, 100.0, -1e4, 1e30, float('nan'), float('nan'), 88.5, float('inf'), -float('inf'),
                             0.0, -0.0])
        pred.view(-1)[idx] = vals
        next_pred.view(-1)[idx.flip(0)] = vals
    traj = None
    if c['traj']:
        traj = done.clone()
        traj.view(-1)[torch.arange(0, done.numel(), 50)[1:] - 1] = True  # truncated trajectories every 50 steps
        traj[-1] = True
        traj = traj.float()
    if c['done'] == 'none':
        done = None
    elif c['done'] == 'float':
        done = done.float()
    mu = torch.randn(1, generator=g) if c['mode'] == 'popart' else None
    sigma = torch.rand(1, generator=g) + 0.5 if c['mode'] == 'popart' else None
    if c['col']:
        pred, next_pred = pred[:, None], next_pred[:, None]
    t = {'pred': pred, 'next_pred': next_pred, 'reward': reward, 'done': done, 'traj_flag': traj, 'mu': mu, 'sigma': sigma}
    return {k: (v.to(device) if v is not None else None) for k, v in t.items()}


def run_oracle(ref, c, t, ieee_sqrt=False):
    return ppof_oracle.ppof_recompute(ref, t['pred'], t['next_pred'], t['reward'], t['done'], t['traj_flag'], GAMMA, LAMBDA,
                                      c['mode'], np.float64(STD), t['mu'], t['sigma'], ieee_sqrt=ieee_sqrt)


def run_ours(c, t):
    data = b2.gae_data(t['pred'], t['next_pred'], t['reward'], t['done'], t['traj_flag'])
    return b2.ppof_gae_returns(data, GAMMA, LAMBDA, c['mode'], std=np.float64(STD) if c['mode'] == 'baseline' else None,
                               popart_mu=t['mu'], popart_sigma=t['sigma'])


def load_fixture(name):
    with np.load(os.path.join(GOLDEN_DIR, name + '.npz'), allow_pickle=False) as z:
        d = {k: z[k] for k in z.files}
    case = json.loads(str(d.pop('case')))
    t = {k: (torch.from_numpy(d['in_' + k]) if 'in_' + k in d else None) for k in INPUTS}
    return case, t, d


def same_bits(got, want, what=''):
    """bit for bit (the sign of a zero included); NaN matches NaN whatever its payload"""
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    ng, nw = np.isnan(got), np.isnan(want)
    ok = np.array_equal(ng, nw) and np.array_equal(got[~ng].view(np.int32), want[~nw].view(np.int32))
    assert ok, (what, ulp_gap(got, want))


def ulp_gap(got, want):
    """largest distance in units in the last place over the elements where both are finite, and the count of mismatched
    non-finite ones"""
    got, want = np.asarray(got, np.float32).reshape(-1), np.asarray(want, np.float32).reshape(-1)
    fin = np.isfinite(got) & np.isfinite(want)

    def ordered(x):
        i = x.view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7fffffff), i)

    gap = int(np.max(np.abs(ordered(got[fin]) - ordered(want[fin])))) if fin.any() else 0
    bad = int(np.sum(~fin & ~((got == want) | (np.isnan(got) & np.isnan(want)))))
    return {'max_ulp': gap, 'nonfinite_mismatch': bad}


def close(got, want, rtol, scale, what=''):
    """|got - want| <= rtol * (|want| + scale) where want is finite, the same inf / NaN pattern elsewhere.  ``scale``: the
    largest finite decoded value -- adv and the return are sums of decoded values, and where those cancel only the decoded
    magnitude bounds what a 1-ulp difference of log / exp leaves behind."""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    assert np.array_equal(np.isnan(got), np.isnan(want)), what
    inf = np.isinf(want)
    assert np.array_equal(got[inf], want[inf]) and not np.isinf(got[~inf]).any(), what
    fin = np.isfinite(want)
    g, w = got[fin], want[fin]
    err = np.abs(g - w) / (np.abs(w) + scale + 1e-30)
    assert err.size == 0 or err.max() <= rtol, (what, float(err.max()))


def decoded_scale(ref, t, mode):
    dec = ref.inv_symlog if mode == 'symlog' else ref.value_inv_transform
    d = torch.cat([dec(t['pred']).reshape(-1), dec(t['next_pred']).reshape(-1)]).double().numpy()
    d = np.abs(d[np.isfinite(d)])
    return float(d.max()) if d.size else 0.0


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
        if want[k] is None:
            assert t[k] is None, k
        else:
            assert t[k].dtype == want[k].dtype and np.array_equal(t[k].numpy(), want[k].numpy(), equal_nan=True), k


def test_fixtures_cover_the_edges():
    modes = {CASES[n]['mode'] for n in CASES}
    assert modes == set(MODES)
    _, t, d = load_fixture('symlog_n400_inf_nan')
    assert np.isinf(d['out_adv']).any() and np.isnan(d['out_adv']).any() and np.isinf(d['out_value']).any()
    _, t, d = load_fixture('popart_n128_col')
    assert t['pred'].shape == (128, 1) and d['out_adv'].shape == (128, 1) and t['reward'].shape == (128, )
    _, t, _ = load_fixture('baseline_n400_bool')
    assert t['done'].dtype == torch.bool and t['done'].any()
    _, t, _ = load_fixture('baseline_n128')
    assert (t['traj_flag'] != t['done']).any()  # segments cut where no episode ends


@pytest.mark.skipif(not HAVE_REF, reason='reference not importable here')
@pytest.mark.parametrize('name', sorted(CASES))
def test_fixture_outputs_are_the_restated_reference(name):
    case, t, d = load_fixture(name)
    adv, value, ret, stats = run_oracle(ref_loader.load(), case, t)
    same_bits(adv.numpy(), d['out_adv'], 'adv')
    same_bits(value.numpy(), d['out_value'], 'value')
    same_bits(ret.numpy(), d['out_return'], 'return_')
    if stats is not None:
        assert np.array_equal(np.array(stats), d['out_stats'], equal_nan=True)


@pytest.mark.skipif(not HAVE_REF, reason='reference not importable here')
def test_restatement_is_pinned_to_the_live_functions():
    """the restatement runs the live functions: the modes that share PPOPolicy's lines agree with that restatement, the
    decoded ones are the live value maps around the live gae, and the inputs survive"""
    from oracle import rl_oracle
    ref = ref_loader.load()
    t = make_inputs(_case(31, 'baseline', (400, )))
    keep = {k: v.clone() for k, v in t.items() if v is not None}
    adv, value, ret, stats = run_oracle(ref, CASES['baseline_n128'], t)
    a2, v2, r2, _, _ = rl_oracle.ppo_policy_gae_returns(t['pred'], t['next_pred'], t['reward'], t['done'], t['traj_flag'],
                                                        GAMMA, LAMBDA, np.float64(STD))
    assert torch.equal(adv, a2) and torch.equal(value, v2) and torch.equal(ret, r2)
    x = ret.numpy()
    assert stats == (float(np.mean(x)), float(np.var(x)), 400.0)  # of the STORED return (ppof.py:206-208)
    for mode, dec, enc in (('value_rescale', ref.value_inv_transform, ref.value_transform),
                           ('symlog', ref.inv_symlog, ref.symlog)):
        adv, value, ret, stats = run_oracle(ref, dict(CASES['baseline_n128'], mode=mode), t)
        v, nv = dec(t['pred']), dec(t['next_pred'])
        want = ref.gae(ref.gae_data(v, nv.clone(), t['reward'], t['done'], t['traj_flag']), GAMMA, LAMBDA)
        assert torch.equal(adv, want) and torch.equal(value, enc(v)) and torch.equal(ret, enc(v + want)) and stats is None
    for k, v in keep.items():
        assert torch.equal(t[k], v), k


@pytest.mark.skipif(not HAVE_REF, reason='reference not importable here')
def test_ieee_restatement_of_value_rescale_is_the_live_pair():
    """h_ieee / h_inv_ieee: the live value_transform / value_inv_transform up to the CPU sqrt's rounding -- the same
    non-finite pattern, equal for most inputs, and within 5e-5 of max(|result|, 1) elsewhere (h^-1 subtracts 1 from a square
    root near 1 and squares the rest, which magnifies a 1-ulp sqrt difference)"""
    ref = ref_loader.load()
    g = torch.Generator().manual_seed(3)
    x = torch.cat([torch.tensor([0.0, -0.0, 1.0, -1.0, float('nan'), float('inf'), -float('inf'), 1e30, -1e-30]),
                   torch.randn(100000, generator=g) * 5, torch.randn(1000, generator=g) * 1e4])
    for mine, live in ((ppof_oracle.h_ieee, ref.value_transform), (ppof_oracle.h_inv_ieee, ref.value_inv_transform)):
        a, b = mine(x).double().numpy(), live(x).double().numpy()
        assert np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(a[np.isinf(b)], b[np.isinf(b)])
        fin = np.isfinite(b)
        assert np.all(np.abs(a[fin] - b[fin]) <= 5e-5 * np.maximum(np.abs(b[fin]), 1.0)), mine.__name__
        assert np.mean(a[fin] == b[fin]) > 0.9


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


# b200rl_gae_returns_norm's arguments by position
_ARG = {'T': 5, 'C': 6, 'mode': 9, 'std': 10, 'mu': 11, 'sigma': 12, 'stats': 16, 'scratch': 18}


@pytest.mark.filterwarnings('ignore:invalid value encountered in cast')  # the stand-in leaves outputs uninitialised
@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('shape', [(400, ), (400, 1), (24576, ), (24577, ), (33, 36)])
def test_marshalling_dry_run(dry, mode, shape):
    c = _case(40, mode, shape[:1] if len(shape) == 2 and shape[1] == 1 else shape, col=len(shape) == 2 and shape[1] == 1)
    t = make_inputs(c)
    out = run_ours(c, t)
    assert [n for n, _ in dry] == ['b200rl_gae_returns_norm']
    a = dry[0][1]
    n = t['reward'].numel()
    T = t['reward'].shape[0]
    assert a[_ARG['T']] == T and a[_ARG['C']] == n // T
    assert a[_ARG['mode']] == MODES.index(mode)
    assert a[_ARG['std']] == (STD if mode == 'baseline' else 0.0)
    assert (a[_ARG['mu']] is not None and a[_ARG['sigma']] is not None) == (mode == 'popart')
    assert (a[_ARG['stats']] is not None) == (mode == 'baseline')
    multi = not (n // T == 1 and T <= 24576)
    assert (a[_ARG['scratch']] is not None) == (multi and mode != 'baseline')
    assert out.adv.shape == out.value.shape == out.return_.shape == t['pred'].shape
    assert (out.return_stats is not None) == (mode == 'baseline') and out.adv_stats.shape == (2, )


@pytest.mark.filterwarnings('ignore:invalid value encountered in cast')
def test_value_maps_dry_run(dry):
    x = torch.randn(7, 3, requires_grad=True)
    y = b2.symlog(x)
    assert [n for n, _ in dry] == ['b200rl_value_map_fwd'] and dry[0][1][0] == 0 and dry[0][1][2] == 21
    y.sum().backward()
    assert [n for n, _ in dry] == ['b200rl_value_map_fwd', 'b200rl_value_map_bwd'] and dry[1][1][0] == 0
    assert x.grad.shape == (7, 3)
    dry.clear()
    b2.inv_symlog(torch.randn(5))
    assert [(n, a[0]) for n, a in dry] == [('b200rl_value_map_fwd', 1)]
    dry.clear()
    assert b2.symlog(torch.zeros(0, 3)).shape == (0, 3) and dry == []  # empty: no launch
    for dt in (torch.float64, torch.float16, torch.bfloat16, torch.int64):
        with pytest.raises(TypeError, match='float32'):
            b2.inv_symlog(torch.zeros(3, dtype=dt))
    assert dry == []


def test_bad_arguments_raise_before_any_call(dry):
    t = make_inputs(_case(41, 'popart', (64, )))
    data = b2.gae_data(t['pred'], t['next_pred'], t['reward'], t['done'], t['traj_flag'])
    with pytest.raises(ValueError, match='value_norm'):
        b2.ppof_gae_returns(data, value_norm='popart_')
    with pytest.raises(ValueError, match='std'):
        b2.ppof_gae_returns(data, value_norm='baseline')
    for std in (0.0, -1.0, float('nan')):
        with pytest.raises(ValueError, match='std'):
            b2.ppof_gae_returns(data, value_norm='baseline', std=std)
    with pytest.raises(ValueError, match='popart_mu'):
        b2.ppof_gae_returns(data, value_norm='popart', popart_mu=t['mu'])
    with pytest.raises(ValueError, match='one float'):
        b2.ppof_gae_returns(data, value_norm='popart', popart_mu=torch.zeros(2), popart_sigma=torch.ones(2))
    with pytest.raises(ValueError, match='shape'):
        b2.ppof_gae_returns(data._replace(value=t['pred'][:-1]), value_norm='symlog')
    with pytest.raises(TypeError, match='float32'):
        b2.ppof_gae_returns(data._replace(value=t['pred'].double()), value_norm='symlog')
    assert dry == []


def test_library_rejects_bad_arguments_before_any_launch():
    """the built library's own checks: they return before any CUDA call, so they run without a device (the pointers are
    never dereferenced)"""
    if not b2.is_built():
        pytest.skip('library not built')
    lib = _lib.load()
    p = 4096  # a non-null stand-in
    ws = 1 << 20

    def call(mode=0, std=1.0, mu=p, sigma=p, T=64, C=1, scratch=None, wsb=ws):
        return lib.b200rl_gae_returns_norm(p, p, p, None, None, T, C, 0.99, 0.95, mode, std, mu, sigma, p, p, p, p, p,
                                           scratch, p, wsb, None)

    assert call(mode=-1) == -1 and call(mode=4) == -1
    assert call(mode=0, std=0.0) == -1 and call(mode=0, std=-2.0) == -1 and call(mode=0, std=float('nan')) == -1
    assert call(mode=3, mu=None) == -1 and call(mode=3, sigma=None) == -1
    for mode in (1, 2, 3):
        assert call(mode=mode, T=33, C=36) == -1  # the decode pass needs its scratch
        assert call(mode=mode, T=24577) == -1
    assert call(T=0) == -1 and call(wsb=ws - 4) == -1
    assert lib.b200rl_value_map_fwd(2, p, 8, p, None) == -1 and lib.b200rl_value_map_bwd(-1, p, p, 8, p, None) == -1
    assert lib.b200rl_value_map_fwd(0, None, 8, p, None) == -1 and lib.b200rl_value_map_bwd(1, p, None, 8, p, None) == -1
    assert lib.b200rl_value_map_fwd(0, None, 0, None, None) == 0  # n == 0: nothing to launch
    assert lib.b200rl_version() >= 109


def test_install_rebinds_ppof_names_and_uninstall_restores(dry, monkeypatch):
    def ref_symlog(x):
        return 'reference'

    def ref_inv_symlog(x):
        return 'reference'

    fake = {}
    for name in ('ding', 'ding.rl_utils', 'ding.rl_utils.value_rescale', 'ding.policy', 'ding.policy.ppof'):
        fake[name] = types.ModuleType(name)
        monkeypatch.setitem(sys.modules, name, fake[name])
    for m in ('ding.rl_utils', 'ding.rl_utils.value_rescale', 'ding.policy.ppof'):
        fake[m].symlog = ref_symlog
        fake[m].inv_symlog = ref_inv_symlog
    done = b2.install()
    for m in ('ding.rl_utils', 'ding.rl_utils.value_rescale', 'ding.policy.ppof'):
        assert (m, 'symlog') in done and (m, 'inv_symlog') in done
        assert fake[m].symlog is b2.rl_utils.symlog and fake[m].inv_symlog is b2.rl_utils.inv_symlog
    b2.uninstall()
    for m in ('ding.rl_utils', 'ding.rl_utils.value_rescale', 'ding.policy.ppof'):
        assert fake[m].symlog is ref_symlog and fake[m].inv_symlog is ref_inv_symlog


# =================================================================================================================
# GPU
# =================================================================================================================
def _check_against(out, want, mode, exact_all):
    adv, value, ret, stats = want
    same_bits(out.adv.cpu().numpy(), adv.cpu().numpy(), 'adv')
    if exact_all:
        same_bits(out.value.cpu().numpy(), value.cpu().numpy(), 'value')
        same_bits(out.return_.cpu().numpy(), ret.cpu().numpy(), 'return_')
    if mode == 'baseline':
        got = out.return_stats.cpu().numpy().astype(np.float64)
        assert np.allclose(got[:2], stats[:2], rtol=2e-6, atol=0, equal_nan=True), (got, stats)
        assert got[2] == stats[2]
    else:
        assert out.return_stats is None
    a = out.adv.cpu().double().numpy().reshape(-1)
    if np.isfinite(a).all() and a.size > 1:
        ast = out.adv_stats.cpu().numpy().astype(np.float64)
        assert np.allclose(ast, [a.mean(), a.std(ddof=1) + 1e-8], rtol=2e-6, atol=1e-7), (ast, a.mean(), a.std(ddof=1))


GPU_SHAPES = [(1, ), (128, ), (400, ), (3200, ), (24576, ), (30000, ), (33, 36), (128, 4096)]


@pytest.mark.gpu
@pytest.mark.skipif(not HAVE_REF, reason='reference not importable here')
@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('shape', GPU_SHAPES, ids=lambda s: 'x'.join(map(str, s)))
def test_semantics_table(mode, shape):
    ref = ref_loader.load()
    c = _case(100 + len(shape) * 7 + shape[0], mode, shape, col=mode == 'popart' and len(shape) == 1)
    t = make_inputs(c)
    if shape == (1, ) and t['traj_flag'] is not None:
        t['traj_flag'][:] = 1.0
    td = {k: (v.cuda() if v is not None else None) for k, v in t.items()}
    keep = {k: v.clone() for k, v in td.items() if v is not None}
    out = run_ours(c, td)
    torch.cuda.synchronize()
    for k, v in keep.items():  # the inputs are only read
        assert torch.equal(td[k], v), k
    assert out.adv.device == td['pred'].device
    cpu = run_oracle(ref, c, t)
    if mode in ('symlog', 'value_rescale'):
        # torch's CPU log / exp and its vectorised CPU sqrt (1 ulp off for some inputs) are not the device's: within 1e-5
        # relative of the live reference on the CPU
        scale = decoded_scale(ref, t, mode)
        for got, want, what in ((out.adv, cpu[0], 'adv'), (out.value, cpu[1], 'value'), (out.return_, cpu[2], 'return_')):
            close(got.cpu().numpy(), want.numpy(), 1e-5, scale, what)
    if mode == 'symlog':  # bit for bit with the reference on the same CUDA tensors
        dev = run_oracle(ref, c, {k: (v.clone() if v is not None else None) for k, v in td.items()})
        _check_against(out, dev, mode, True)
    elif mode == 'value_rescale':  # bit for bit with the reference's lines rounded as IEEE fp32 (true division, IEEE sqrt)
        _check_against(out, run_oracle(ref, c, t, ieee_sqrt=True), mode, True)
    else:
        _check_against(out, cpu, mode, True)
        if mode in ('baseline', 'popart'):  # the device reference multiplies by 1 / std: adv is still bit-exact
            dev = run_oracle(ref, c, {k: (v.clone() if v is not None else None) for k, v in td.items()})
            same_bits(out.adv.cpu().numpy(), dev[0].cpu().numpy(), 'adv vs device reference')


@pytest.mark.gpu
@pytest.mark.parametrize('name', sorted(CASES))
def test_fixtures_on_gpu(name):
    case, t, d = load_fixture(name)
    out = run_ours(case, {k: (v.cuda() if v is not None else None) for k, v in t.items()})
    if case['mode'] in ('symlog', 'value_rescale'):  # CPU log / exp / sqrt: see test_semantics_table
        scale = decoded_scale(ref_loader.load(), t, case['mode']) if HAVE_REF else float(np.nanmax(np.abs(d['out_adv'][
            np.isfinite(d['out_adv'])])))
        for k, what in (('out_adv', 'adv'), ('out_value', 'value'), ('out_return', 'return_')):
            close(getattr(out, what).cpu().numpy(), d[k], 1e-5, scale, what)
    else:
        same_bits(out.adv.cpu().numpy(), d['out_adv'], 'adv')
        same_bits(out.value.cpu().numpy(), d['out_value'], 'value')
        same_bits(out.return_.cpu().numpy(), d['out_return'], 'return_')
    if case['mode'] == 'baseline':
        assert np.allclose(out.return_stats.cpu().numpy().astype(np.float64)[:2], d['out_stats'][:2], rtol=2e-6,
                           equal_nan=True)


@pytest.mark.gpu
def test_host_tensors_are_staged_and_returned_on_the_host():
    c = CASES['value_rescale_n128']
    t = make_inputs(c)
    out = run_ours(c, t)
    assert out.adv.device.type == 'cpu' and out.adv_stats.device.type == 'cpu'
    want = run_ours(c, {k: (v.cuda() if v is not None else None) for k, v in t.items()})
    for a, b in zip(out, want):
        if a is not None:
            assert torch.equal(a, b.cpu())


def _kernels(fn):
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and 'Memcpy' not in e.name
            and 'Memset' not in e.name]


@pytest.mark.gpu
@pytest.mark.parametrize('mode', MODES)
def test_launch_sequence(mode):
    """1-D up to 24576 steps: ONE launch; (T, B): decode pass (none for baseline), the streaming scan, the epilogue"""
    for shape, want in (((400, ), ['gae_seq_kernel']), ((128, 64), ['value_map_kernel', 'gae_ws_kernel', 'returns_kernel'])):
        c = _case(60, mode, shape)
        t = {k: (v.cuda() if v is not None else None) for k, v in make_inputs(c).items()}
        names = _kernels(lambda: run_ours(c, t))
        if mode == 'baseline' and len(shape) == 2:
            want = want[1:]
        assert len(names) == len(want) and all(w in n for w, n in zip(want, names)), names


EDGES = [0.0, -0.0, 1.0, -1.0, float('inf'), -float('inf'), float('nan'), 1e30, -1e30, 88.5, 88.8, 89.0, -89.0, 100.0,
         -100.0, 1e-30, -1e-45, 3.4e38]


@pytest.mark.gpu
@pytest.mark.skipif(not HAVE_REF, reason='reference not importable here')
@pytest.mark.parametrize('name', ['symlog', 'inv_symlog'])
def test_value_maps_against_the_reference_on_the_device(name):
    ref = ref_loader.load()
    g = torch.Generator().manual_seed(5)
    base = torch.cat([torch.tensor(EDGES), torch.randn(5000, generator=g) * 10, torch.randn(3, 7, generator=g).reshape(-1)])
    up = torch.randn(base.numel(), generator=g)
    up[:4] = torch.tensor([-1.0, 2.0, -0.0, 0.0])
    n = base.numel()
    for shape in ((n, ), (n // 3, 3)):
        x0 = base[:int(np.prod(shape))].reshape(shape).cuda()
        gy = up[:x0.numel()].reshape(shape).cuda()
        xa = x0.clone().requires_grad_(True)
        xb = x0.clone().requires_grad_(True)
        ya = getattr(b2, name)(xa)
        yb = getattr(ref, name)(xb)
        same_bits(ya.detach().cpu().numpy(), yb.detach().cpu().numpy(), name)
        ya.backward(gy)
        yb.backward(gy)
        same_bits(xa.grad.cpu().numpy(), xb.grad.cpu().numpy(), name + ' grad')
    e = torch.zeros(0, device='cuda', requires_grad=True)
    y = getattr(b2, name)(e)
    assert y.shape == (0, )
    y.sum().backward()
    assert e.grad.shape == (0, )
    xc = base[:64].clone().requires_grad_(True)  # a host tensor: staged to the device, returned on the host
    yc = getattr(b2, name)(xc)
    assert yc.device.type == 'cpu'
    same_bits(yc.detach().numpy(), getattr(b2, name)(base[:64].cuda()).cpu().numpy(), name + ' host')
    yc.backward(up[:64])
    assert xc.grad is not None and xc.grad.device.type == 'cpu'


@pytest.mark.gpu
@pytest.mark.skipif(not HAVE_REF, reason='reference not importable here')
def test_install_routes_ppof_names_to_the_kernel():
    """a module holding PPOF's imported names (ppof.py:11-13) calls the kernel after install()"""
    ref = ref_loader.load()
    policy = types.ModuleType('ding.policy.fake_ppof_for_install_test')
    for n in ('gae', 'gae_data', 'value_transform', 'value_inv_transform', 'symlog', 'inv_symlog'):
        setattr(policy, n, getattr(ref, n))
    sys.modules[policy.__name__] = policy
    try:
        b2.install()
        assert policy.symlog is b2.rl_utils.symlog and policy.inv_symlog is b2.rl_utils.inv_symlog
        assert ref.symlog is b2.rl_utils.symlog
        x = torch.randn(257, device='cuda') * 5
        names = _kernels(lambda: policy.symlog(policy.inv_symlog(x)))
        assert len(names) == 2 and all('value_map_kernel' in n for n in names), names
    finally:
        b2.uninstall()
        del sys.modules[policy.__name__]
    assert ref.symlog is not b2.rl_utils.symlog
