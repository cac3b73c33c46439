"""torch.compile over the functions that reach ``b200rl`` custom ops beyond the plugin-boundary eight and the language-model
losses: the quantile TD losses (QR-DQN, IQN, FQF), the continuous-action PPO losses, symlog / inv_symlog, the advantage
recomputes (gae_returns, ppof_gae_returns, normalize_advantage, ppo_error_adv_norm), and the siblings that share the
staging code of a traced operator (q_1step / v_1step / v_nstep / bdq_nstep / dist_1step TD, ppo_policy_error, the discrete
HAPPO losses).

CPU part: against the logging stand-in for the CUDA library of ``tests/test_launch_log.py``, each function compiles with
``backend='aot_eager', fullgraph=True`` and its compiled forward + backward makes the launches of the eager call, apart
from the differences named per case; every error the eager call raises on bad input is raised while compiling; every op
schema holds tensors and scalars only; and every function of ``TRACED`` has a case.

GPU part: ``torch.library.opcheck`` on every new op; inductor results bit-identical to eager and within the suites'
tolerances of the reference, on the cases of ``tests/cases.py`` and the golden sets ``tests/golden/{pg_continuous,ppof}``;
``mode="reduce-overhead"`` replays; a dynamic batch without recompiling; three small learner steps, model included, that
compile without a graph break.
"""
import numpy as np
import pytest
import torch
import torch._dynamo

import di_engine_b200 as b2
from di_engine_b200 import ops
from tests import cases, test_pg_continuous as pg_continuous, test_ppof as ppof
from tests.test_compile import _launches, _queries, _same_record, _stand_in
from tests.test_launch_log import _cont_inputs, _q_inputs

api = b2.rl_utils
B, N, D, NSTEP, T = 4, 5, 3, 3, 6

# the public functions this file compiles: the ones whose calls reach the custom ops below, and the siblings that share the
# staging code of an op traced since the plugin-boundary eight.  INTEGRATION.md section 3d lists the rebound functions
# that still end in an autograd.Function and so still break the graph; they are not tested here.
TRACED = ('qrdqn_nstep_td_error', 'iqn_nstep_td_error', 'fqf_nstep_td_error', 'ppo_error_continuous',
          'ppo_policy_error_continuous', 'happo_error_continuous', 'happo_policy_error_continuous', 'symlog', 'inv_symlog',
          'gae_returns', 'ppof_gae_returns', 'normalize_advantage', 'ppo_error_adv_norm', 'q_1step_td_error',
          'v_1step_td_error', 'v_nstep_td_error', 'bdq_nstep_td_error', 'dist_1step_td_error', 'ppo_policy_error',
          'happo_error', 'happo_policy_error')
NEW_OPS = ('gae_returns', 'gae_returns_norm', 'adv_stats', 'normalize', 'value_map', 'value_map_bwd', 'quantile_fwd',
           'quantile_bwd', 'ppoc_loss', 'ppoc_bwd')


@pytest.fixture(autouse=True)
def _distribution_validation():
    """dynamo turns off torch.distributions' argument validation for the whole process the first time it runs"""
    validate = torch.distributions.Distribution._validate_args
    yield
    torch.distributions.Distribution.set_default_validate_args(validate)


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _rg(t):
    return t.requires_grad_(True)


def _loss_only(r):
    """(loss, td_error_per_sample) -> loss, the per-sample error leaving detached, as a learner takes it for priorities"""
    return (r[0], ) if isinstance(r, tuple) else (r, )


# ---------------------------------------------------------------------------------------------------------------------
# the cases: name -> (inputs(g) -> args, fn(*args) -> the differentiable outputs to back-propagate, or None)
# ---------------------------------------------------------------------------------------------------------------------
def _quantile_in(kind):
    def inputs(g):
        if kind == 'qrdqn':
            q, nq, act, nact, reward, done = _q_inputs(g, (B, N, 3))
            return api.qrdqn_nstep_td_data(q, nq, act, nact, reward, done, torch.rand(B, 3, 1, generator=g), None),
        if kind == 'iqn':
            q, nq, act, nact, reward, done = _q_inputs(g, (3, B, N))
            return api.iqn_nstep_td_data(q, nq, act, nact, reward, done, torch.rand(3, B, 1, generator=g), None),
        q, nq, act, nact, reward, done = _q_inputs(g, (B, 3, N))
        return api.fqf_nstep_td_data(q, nq, act, nact, reward, done, torch.rand(B, 3, generator=g), None),
    return inputs


def _quantile_fn(kind, **kw):
    fn = getattr(api, kind + '_nstep_td_error')
    return lambda data: _loss_only(fn(data, 0.95, nstep=NSTEP, **kw))


def _ppoc_in(policy_only, hetero=False):
    def inputs(g):
        new, old, act, vn, vo, adv, ret, factor = _cont_inputs(g)
        if hetero:
            if policy_only:
                return (new, old, act, adv, None),
            return api.happo_data(new, old, act, vn, vo, adv, ret, None, factor),
        if policy_only:
            return api.ppo_policy_data_continuous(new, old, act, adv, None, None),
        return api.ppo_data(new, old, act, vn, vo, adv, ret, None, None),
    return inputs


def _ppoc_fn(name):
    fn = getattr(api, name)
    return lambda data: tuple(x for x in fn(data)[0] if isinstance(x, torch.Tensor))


def _ppo_in(policy_only, hetero=False):
    def inputs(g):
        ln, lo = _rg(torch.randn(B, N, generator=g)), torch.randn(B, N, generator=g)
        act = torch.randint(0, N, (B, ), generator=g)
        vn = _rg(torch.randn(B, generator=g))
        vo, adv, ret = (torch.randn(B, generator=g) for _ in range(3))
        factor = torch.rand(B, 1, generator=g)
        if policy_only:
            return (api.happo_policy_data(ln, lo, act, adv, None, factor) if hetero else
                    api.ppo_policy_data(ln, lo, act, adv, None, None)),
        return (api.happo_data(ln, lo, act, vn, vo, adv, ret, None, factor) if hetero else
                api.ppo_data(ln, lo, act, vn, vo, adv, ret, None, None)),
    return inputs


def _gae_in(one_d=False):
    def inputs(g):
        shape = (T * B, ) if one_d else (T, B)
        v, nv, r = (torch.randn(*shape, generator=g) for _ in range(3))
        done = (torch.rand(*shape, generator=g) < 0.2).float()
        return api.gae_data(v, nv, r, done, done.clone()),
    return inputs


def _ppof_fn(mode):
    extra = {'baseline': {'std': 1.7}, 'popart': {'popart_mu': torch.tensor([0.3]), 'popart_sigma': torch.tensor([2.0])}}

    def fn(data):
        return None, api.ppof_gae_returns(data, 0.99, 0.95, value_norm=mode, **extra.get(mode, {}))
    return fn


def _v1_in(g):
    v, nv = _rg(torch.randn(B, generator=g)), torch.randn(B, generator=g)
    return api.v_1step_td_data(v, nv, torch.randn(B, generator=g), (torch.rand(B, generator=g) < 0.3).float(), None),


def _vn_in(g):
    v, nv = _rg(torch.randn(B, generator=g)), torch.randn(B, generator=g)
    return api.v_nstep_td_data(v, nv, torch.randn(NSTEP, B, generator=g), (torch.rand(B, generator=g) < 0.3).float(),
                               None, None),


def _q1_in(g):
    q, nq, act, nact, reward, done = _q_inputs(g, (B, N))
    return api.q_1step_td_data(q, nq, act, nact, reward[0], done, None),


def _bdq_in(g):
    q, nq, act, nact, reward, done = _q_inputs(g, (B, D, N), (B, D))
    return api.q_nstep_td_data(q, nq, act, nact, reward, done, None),


def _d1_in(g):
    dist = _rg(torch.rand(B, N, 11, generator=g) + 0.1)
    act, nact = torch.randint(0, N, (B, ), generator=g), torch.randint(0, N, (B, ), generator=g)
    return api.dist_1step_td_data(dist, torch.rand(B, N, 11, generator=g) + 0.1, act, nact, torch.randn(B, generator=g),
                                  (torch.rand(B, generator=g) < 0.3).float(), None),


def _symlog_in(g):
    return _rg(torch.randn(B, N, generator=g) * 3),


def _adv_in(g):
    return torch.randn(T, B, generator=g),


CASES = {
    'qrdqn_nstep_td_error': (_quantile_in('qrdqn'), _quantile_fn('qrdqn')),
    'qrdqn_nstep_td_error[value_gamma]': (_quantile_in('qrdqn'), _quantile_fn('qrdqn', value_gamma=0.9)),
    'iqn_nstep_td_error': (_quantile_in('iqn'), _quantile_fn('iqn', kappa=0.7)),
    'fqf_nstep_td_error': (_quantile_in('fqf'), _quantile_fn('fqf')),
    'ppo_error_continuous': (_ppoc_in(False), _ppoc_fn('ppo_error_continuous')),
    'ppo_policy_error_continuous': (_ppoc_in(True), _ppoc_fn('ppo_policy_error_continuous')),
    'happo_error_continuous': (_ppoc_in(False, True), _ppoc_fn('happo_error_continuous')),
    'happo_policy_error_continuous': (_ppoc_in(True, True), _ppoc_fn('happo_policy_error_continuous')),
    'symlog': (_symlog_in, lambda x: (api.symlog(x).sum(), )),
    'inv_symlog': (_symlog_in, lambda x: (api.inv_symlog(x * 0.3).sum(), )),
    'gae_returns': (_gae_in(True), lambda data: (None, api.gae_returns(data, 0.99, 0.95))),
    'gae_returns[value_norm]': (_gae_in(), lambda data: (None, api.gae_returns(data, 0.99, 0.95, value_norm_std=1.3))),
    'ppof_gae_returns[baseline]': (_gae_in(True), _ppof_fn('baseline')),
    'ppof_gae_returns[value_rescale]': (_gae_in(), _ppof_fn('value_rescale')),
    'ppof_gae_returns[symlog]': (_gae_in(True), _ppof_fn('symlog')),
    'ppof_gae_returns[popart]': (_gae_in(), _ppof_fn('popart')),
    'normalize_advantage': (_adv_in, lambda adv: (None, api.normalize_advantage(adv))),
    'ppo_error_adv_norm': (_ppo_in(False), lambda data: tuple(api.ppo_error_adv_norm(data)[0][:3])),
    'q_1step_td_error': (_q1_in, lambda data: _loss_only(api.q_1step_td_error(data, 0.95))),
    'v_1step_td_error': (_v1_in, lambda data: _loss_only(api.v_1step_td_error(data, 0.99))),
    'v_nstep_td_error': (_vn_in, lambda data: _loss_only(api.v_nstep_td_error(data, 0.99, NSTEP))),
    'bdq_nstep_td_error': (_bdq_in, lambda data: _loss_only(api.bdq_nstep_td_error(data, 0.95, nstep=NSTEP))),
    'dist_1step_td_error': (_d1_in, lambda data: _loss_only(api.dist_1step_td_error(data, 0.95, -10.0, 10.0, 11))),
    'ppo_policy_error': (_ppo_in(True), lambda data: tuple(api.ppo_policy_error(data)[0][:2])),
    'happo_error': (_ppo_in(False, True), lambda data: tuple(api.happo_error(data)[0][:3])),
    'happo_policy_error': (_ppo_in(True, True), lambda data: tuple(api.happo_policy_error(data)[0][:2])),
}
MIX = (1.0, 0.5, -0.01, 0.3)


def _upstream_as_one_vector(launches):
    """ppo_error_continuous's verify launch: the op hands the four upstream gradients over as one vector, so a loss that
    does not reach an output passes a pointer to 0 where the autograd.Function passed a null pointer (both read as 0)"""
    out = []
    for fn, check, args in launches:
        if check == 'b200rl_ppo_continuous_fwd_grad(verify)':
            args = args[:21] + [False] * 4 + args[25:]
        out.append((fn, check, args))
    return out


# the named differences between the eager and the compiled launch sequence, per case
DIFFERENCES = {name: _upstream_as_one_vector for name in CASES if name.startswith(('ppo_error_cont', 'ppo_policy_error_cont',
                                                                                    'happo_error_cont', 'happo_policy_error_cont'))}


def _run(fn, name, seed=7):
    inputs, _ = CASES[name]
    args = inputs(_g(seed))
    with _stand_in() as log:
        outs = fn(*args)
        diff = [o for o in outs if isinstance(o, torch.Tensor) and o.requires_grad]
        if diff:
            sum(w * o for w, o in zip(MIX, diff)).backward()
    return log


def test_every_traced_function_has_a_case():
    public = set(api.HOT_PATH_FUNCTIONS) | {'gae_returns', 'ppof_gae_returns', 'normalize_advantage', 'ppo_error_adv_norm'}
    assert set(TRACED) <= public
    assert sorted(set(TRACED) - {name.split('[')[0] for name in CASES}) == []


@pytest.mark.filterwarnings('ignore:invalid value encountered in cast')  # the stand-in leaves outputs uninitialised
@pytest.mark.parametrize('name', sorted(CASES))
def test_compiled_launch_sequence_matches_eager(name):
    fn = CASES[name][1]
    torch._dynamo.reset()
    want = _run(fn, name)
    got = _run(torch.compile(fn, backend='aot_eager', fullgraph=True), name)
    assert len(want) > 0
    assert _launches(got) == DIFFERENCES.get(name, lambda x: x)(_launches(want))
    # the backward op of ppo_policy_error / happo repeats the forward's *_supported query (tests/test_compile.py)
    assert _queries(got) == _queries(want) * (2 if _queries(want) else 1)


def _bad_inputs():
    g = _g(3)
    q, nq, act, nact, reward, done = _q_inputs(g, (B, N, 3))
    new, old, cact, vn, vo, adv, ret, _ = _cont_inputs(g)
    gd = _gae_in()(g)[0]
    ln, lo = torch.randn(B, N, generator=g), torch.randn(B, N, generator=g)
    pact, pvn = torch.randint(0, N, (B, ), generator=g), torch.randn(B, generator=g)
    return {
        'qrdqn_nstep_td_error': (ValueError, lambda: api.qrdqn_nstep_td_error(
            api.qrdqn_nstep_td_data(q, nq[:, :2], act, nact, reward, done, 3, None), 0.95, nstep=NSTEP)),
        'qrdqn_nstep_td_error[weight]': (ValueError, lambda: api.qrdqn_nstep_td_error(
            api.qrdqn_nstep_td_data(q, nq, act, nact, reward, done, 3, torch.ones(B + 1)), 0.95, nstep=NSTEP)),
        'iqn_nstep_td_error[value_gamma]': (ValueError, lambda: api.iqn_nstep_td_error(
            api.iqn_nstep_td_data(q.permute(2, 0, 1), nq.permute(2, 0, 1), act, nact, reward, done, torch.rand(3, B, 1),
                                  None), 0.95, nstep=NSTEP, value_gamma=torch.ones(B + 2))),
        'ppo_error_continuous': (ValueError, lambda: api.ppo_error_continuous(
            api.ppo_data(new, old, cact, vn[:2], vo, adv, ret, None, None))),
        'ppo_error_continuous[kl_type]': (ValueError, lambda: api.ppo_error_continuous(
            api.ppo_data(new, old, cact, vn, vo, adv, ret, None, old), kl_type='k9')),
        'ppo_policy_error_continuous[dual_clip]': (AssertionError, lambda: api.ppo_policy_error_continuous(
            api.ppo_policy_data_continuous(new, old, cact, adv, None, None), dual_clip=0.5)),
        'symlog': (TypeError, lambda: api.symlog(torch.randn(3, dtype=torch.float64))),
        'gae_returns': (ValueError, lambda: api.gae_returns(gd._replace(next_value=gd.next_value[:2]))),
        'ppof_gae_returns[value_norm]': (ValueError, lambda: api.ppof_gae_returns(gd, value_norm='minmax')),
        'ppof_gae_returns[std]': (ValueError, lambda: api.ppof_gae_returns(gd, value_norm='baseline', std=0.0)),
        'ppof_gae_returns[popart]': (ValueError, lambda: api.ppof_gae_returns(gd, value_norm='popart')),
        'normalize_advantage': (TypeError, lambda: api.normalize_advantage(torch.randn(4, dtype=torch.float64))),
        'ppo_error_adv_norm': (ValueError, lambda: api.ppo_error_adv_norm(
            api.ppo_data(ln, lo, pact, pvn, pvn, pvn, pvn, None, None), adv_stats=torch.ones(3))),
    }


@pytest.mark.parametrize('name', sorted(_bad_inputs()))
def test_eager_errors_are_raised_while_compiling(name):
    exc, call = _bad_inputs()[name]
    torch._dynamo.reset()
    with _stand_in():
        with pytest.raises(exc) as eager:
            call()
        # dynamo stops tracing at the raise and runs the frame as Python, which raises what eager mode raises
        with pytest.raises(exc) as compiled:
            torch.compile(call, backend='aot_eager')()
    assert str(compiled.value) == str(eager.value)


def test_new_ops_schemas_hold_only_tensors_and_scalars():
    for name in NEW_OPS:
        schema = getattr(torch.ops.b200rl, name).default._schema
        for a in schema.arguments:
            assert str(a.type) in ('Tensor', 'Optional[Tensor]', 'SymInt', 'int', 'float', 'Optional[float]', 'bool', 'str'), (
                name, a.name, a.type)


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def _cuda(x):
    if isinstance(x, torch.Tensor):
        return x.detach().cuda().requires_grad_(x.requires_grad)
    if isinstance(x, dict):
        return {k: _cuda(v) for k, v in x.items()}
    if isinstance(x, tuple):
        items = [_cuda(y) for y in x]
        return type(x)(*items) if hasattr(x, '_fields') else tuple(items)
    return x


def _recording():
    from torch.utils._python_dispatch import TorchDispatchMode
    calls = []

    class Record(TorchDispatchMode):

        def __torch_dispatch__(self, func, types, args=(), kwargs=None):
            if func.namespace == 'b200rl':
                calls.append((func, args, kwargs or {}))
            return func(*args, **(kwargs or {}))

    return Record(), calls


OPCHECK_CASES = ('qrdqn_nstep_td_error', 'qrdqn_nstep_td_error[value_gamma]', 'iqn_nstep_td_error', 'fqf_nstep_td_error',
                 'ppo_error_continuous', 'happo_policy_error_continuous', 'symlog', 'inv_symlog', 'gae_returns',
                 'gae_returns[value_norm]', 'ppof_gae_returns[baseline]', 'ppof_gae_returns[popart]',
                 'normalize_advantage')


@pytest.mark.gpu
@pytest.mark.parametrize('name', OPCHECK_CASES)
def test_opcheck(name):
    inputs, fn = CASES[name]
    args = _cuda(inputs(_g(11)))
    mode, calls = _recording()
    with mode, pytest.MonkeyPatch.context() as mp:
        mp.setattr(torch.compiler, 'is_compiling', lambda: True)  # the traced path, run eagerly
        mp.setattr(api.ppo, 'LAZY_INFO', True)
        if name.startswith('ppof'):  # popart's mu / sigma were made on the host
            mp.setattr(ops, 'to_device', lambda t, dev: t.to(dev) if isinstance(t, torch.Tensor) else t)
        outs = fn(*args)
        diff = [o for o in outs if isinstance(o, torch.Tensor) and o.requires_grad]
        if diff:
            sum(w * o for w, o in zip(MIX, diff)).backward()
    seen = set()
    for op, a, k in calls:
        if op in seen:
            continue
        seen.add(op)
        if op._opname.endswith('_bwd'):  # a backward op is not differentiated again
            a, k = torch.utils._pytree.tree_map_only(torch.Tensor, lambda x: x.detach(), (a, k))
        # each call gets the initial upstream-gradient record, so that its outputs are a function of its inputs
        with pytest.MonkeyPatch.context() as mp:
            mp.setattr(ops, 'ppo_hint', lambda dev, kind='ppo': torch.tensor(ops._HINT_INIT[kind], device=dev))
            torch.library.opcheck(op, a, k)
    assert {op._opname for op in seen} & set(NEW_OPS)


class _CompiledAPI:
    """The reference's names, with the functions of the GPU cases compiled (inductor, fullgraph); td_error_per_sample
    leaves the graph detached, and the PPO monitors are read after the call (``LAZY_INFO``), as in tests/test_compile.py"""
    TD = ('qrdqn_nstep_td_error', 'iqn_nstep_td_error', 'fqf_nstep_td_error', 'v_1step_td_error', 'v_nstep_td_error',
          'bdq_nstep_td_error')
    PLAIN = ('q_1step_td_error', 'dist_1step_td_error')
    LAZY = ('ppo_error_continuous', 'ppo_policy_error', 'happo_error')

    def __init__(self, **kw):
        for name in self.TD:
            f = getattr(api, name)
            setattr(self, name, torch.compile(lambda *a, _f=f, **k: (lambda l, p: (l, p.detach()))(*_f(*a, **k)),
                                              fullgraph=True, **kw))
        for name in self.PLAIN:
            setattr(self, name, torch.compile(getattr(api, name), fullgraph=True, **kw))
        for name in self.LAZY:
            setattr(self, name, self._lazy(torch.compile(getattr(api, name), fullgraph=True, **kw)))

    @staticmethod
    def _lazy(compiled):
        def call(*a, **k):
            lazy, api.ppo.LAZY_INFO = api.ppo.LAZY_INFO, True
            try:
                loss, info = compiled(*a, **k)
            finally:
                api.ppo.LAZY_INFO = lazy
            return loss, type(info)(*(float(x) for x in info))
        return call

    def __getattr__(self, name):
        return getattr(api, name)


GPU_CASES = ('ppoc_basic', 'ppoc_w_dc_novc', 'ppoc_kl_k3', 'ppoc_old_1d', 'qrdqn_basic', 'qrdqn_w_vg', 'qrdqn_scalar_tau',
             'iqn_basic', 'iqn_w_kappa', 'fqf_basic', 'fqf_w_kappa', 'q1td_basic', 'q1td_w', 'v1td_basic', 'v1td_w_nodone',
             'v1td_2d', 'vntd_n3', 'vntd_n5_w_vg', 'bdq_n3', 'bdq_n5_w_vg', 'bdq_cum', 'd1td_basic', 'd1td_marl',
             'ppo_policy_basic', 'ppo_policy_w_dc_kl', 'happo_basic', 'happo_marl')


@pytest.mark.gpu
@pytest.mark.parametrize('name', GPU_CASES)
def test_inductor_bit_identical_to_eager_and_within_reference_tolerance(name):
    from oracle import rl_oracle
    torch._dynamo.reset()
    compiled = _CompiledAPI()
    op, t, p = cases.build_cases()[name]
    with _same_record() as restore:
        want = cases.run_api(api, op, t, p, device='cuda:0')
        restore()
        got = cases.run_api(compiled, op, t, p, device='cuda:0')
    cases.compare(got, want, exact=True)
    cases.compare(got, cases.run_oracle(rl_oracle, op, t, p), rtol=1e-5, atol=1e-5)


def _outputs(outs, args):
    """every tensor a call returned, then the gradients of its differentiable inputs"""
    flat = [x for x in torch.utils._pytree.tree_leaves(outs) if isinstance(x, torch.Tensor)]
    res = [x.detach().clone() for x in flat]
    diff = [o for o in outs if isinstance(o, torch.Tensor) and o.requires_grad]
    if diff:
        leaves = [x for x in torch.utils._pytree.tree_leaves(args) if isinstance(x, torch.Tensor) and x.requires_grad]
        res += [g.clone() for g in torch.autograd.grad(sum(w * o for w, o in zip(MIX, diff)), leaves)]
    return res


@pytest.mark.gpu
@pytest.mark.parametrize('name', ('ppof_gae_returns[baseline]', 'ppof_gae_returns[symlog]', 'gae_returns[value_norm]',
                                  'normalize_advantage', 'ppo_error_adv_norm', 'happo_error_continuous', 'inv_symlog'))
def test_inductor_bit_identical_to_eager(name, monkeypatch):
    monkeypatch.setattr(api.ppo, 'LAZY_INFO', True)
    inputs, fn = CASES[name]
    torch._dynamo.reset()
    compiled = torch.compile(fn, fullgraph=True)
    for seed in (21, 22):
        with _same_record() as restore:
            args = _cuda(inputs(_g(seed)))
            want = _outputs(fn(*args), args)
            restore()
            args = _cuda(inputs(_g(seed)))
            got = _outputs(compiled(*args), args)
        assert len(got) == len(want)
        for a, b in zip(got, want):
            assert torch.equal(a, b), name


@pytest.mark.gpu
@pytest.mark.parametrize('name', ('qrdqn_nstep_td_error[value_gamma]', 'ppo_error_continuous', 'symlog',
                                  'ppof_gae_returns[symlog]'))
def test_reduce_overhead_replays_bit_identical_to_eager(name, monkeypatch):
    monkeypatch.setattr(api.ppo, 'LAZY_INFO', True)
    # no workspace, record or constant exists yet: the compiled call's warm-up is the first to need them
    for k in ('_WS', '_HINT', '_CONST'):
        monkeypatch.setattr(ops, k, {})
    inputs, fn = CASES[name]
    torch._dynamo.reset()
    compiled = torch.compile(fn, mode='reduce-overhead', fullgraph=True)
    allocated = []
    lasting = ops.lasting
    monkeypatch.setattr(ops, 'lasting', lambda make, dev: allocated.append(dev) or lasting(make, dev))
    for step in range(12):  # 2 warm-up / record calls, then 10 replays
        with _same_record() as restore:
            args = _cuda(inputs(_g(100 + step)))
            got = _outputs(compiled(*args), args)
            restore()
            args = _cuda(inputs(_g(100 + step)))
            want = _outputs(fn(*args), args)
        for a, b in zip(got, want):
            assert torch.equal(a, b), (name, step)
        if step == 1:
            allocated.clear()
    assert allocated == [], 'a workspace, record or constant was allocated after warm-up'


@pytest.mark.gpu
@pytest.mark.parametrize('name', ('qrdqn_nstep_td_error', 'ppo_error_continuous'))
def test_dynamic_batch_does_not_recompile(name, monkeypatch):
    from torch._dynamo.utils import counters
    monkeypatch.setattr(api.ppo, 'LAZY_INFO', True)
    torch._dynamo.reset()
    counters.clear()
    fn = torch.compile(CASES[name][1], fullgraph=True)

    def args(S, seed):
        g = _g(seed)
        if name == 'ppo_error_continuous':
            mu, sigma = (torch.randn(S, 3, generator=g).cuda(), (torch.rand(S, 3, generator=g) + 0.5).cuda())
            mo, so, act = torch.randn(S, 3, generator=g).cuda(), (torch.rand(S, 3, generator=g) + 0.5).cuda(), \
                torch.randn(S, 3, generator=g).cuda()
            vn, vo, adv, ret = (torch.randn(S, generator=g).cuda() for _ in range(4))
            ts = [mu, sigma, mo, so, act, vn, vo, adv, ret]
            for t in ts:
                torch._dynamo.mark_dynamic(t, 0)
            mu.requires_grad_(True), sigma.requires_grad_(True), vn.requires_grad_(True)
            return (api.ppo_data({'mu': mu, 'sigma': sigma}, {'mu': mo, 'sigma': so}, act, vn, vo, adv, ret, None, None), )
        q, nq = torch.randn(S, 6, 8, generator=g).cuda(), torch.randn(S, 6, 8, generator=g).cuda()
        act, nact = torch.randint(0, 6, (S, ), generator=g).cuda(), torch.randint(0, 6, (S, ), generator=g).cuda()
        reward, done = torch.randn(3, S, generator=g).cuda(), (torch.rand(S, generator=g) < 0.2).float().cuda()
        tau = torch.rand(S, 8, 1, generator=g).cuda()
        for i, t in enumerate((q, nq, act, nact, reward, done, tau)):
            torch._dynamo.mark_dynamic(t, 1 if i == 4 else 0)
        q.requires_grad_(True)
        return (api.qrdqn_nstep_td_data(q, nq, act, nact, reward, done, tau, None), )

    for S in (64, 320):
        a = args(S, S)
        with _same_record() as restore:
            want = CASES[name][1](*a)
            restore()
            got = fn(*a)
        assert torch.equal(got[0], want[0])
    assert counters['stats']['unique_graphs'] == 1, dict(counters['stats'])


def _bits(x):
    """the bit patterns of a float32 array, so that NaN compares equal to the same NaN"""
    return np.ascontiguousarray(np.asarray(x, np.float32)).view(np.uint32)


PG_FIXTURES = [n for n in pg_continuous.fixture_names() if n.startswith('ppo_')]


@pytest.mark.gpu
@pytest.mark.parametrize('name', PG_FIXTURES)
def test_pg_continuous_fixtures_compiled(name):
    """ppo_policy_error_continuous on the golden set of tests/test_pg_continuous.py, compiled: bit-identical to eager and
    within that suite's tolerance of the stored reference outputs and gradients"""
    case, t, want = pg_continuous.load_fixture(name)
    torch._dynamo.reset()
    compiled = _CompiledAPI()
    compiled.ppo_policy_error_continuous = compiled._lazy(torch.compile(api.ppo_policy_error_continuous, fullgraph=True))
    with _same_record() as restore:
        eager = pg_continuous.run(api, case, t, 'cuda')
        restore()
        got = pg_continuous.run(compiled, case, t, 'cuda')
    assert set(got) == set(eager)
    for k in eager:
        assert np.array_equal(_bits(got[k]), _bits(eager[k])), k
    pg_continuous.compare(got, want)


@pytest.mark.gpu
@pytest.mark.parametrize('name', sorted(ppof.CASES))
def test_ppof_fixtures_compiled(name):
    """ppof_gae_returns on the golden set of tests/test_ppof.py, compiled: bit-identical to eager, and bit-identical to the
    stored outputs where that suite requires it ('baseline', 'popart'); within its tolerance otherwise"""
    case, t, d = ppof.load_fixture(name)
    t = {k: (v.cuda() if v is not None else None) for k, v in t.items()}
    std = float(ppof.STD) if case['mode'] == 'baseline' else None

    def call(pred, next_pred, reward, done, traj_flag, mu, sigma):
        return api.ppof_gae_returns(api.gae_data(pred, next_pred, reward, done, traj_flag), ppof.GAMMA, ppof.LAMBDA,
                                    case['mode'], std=std, popart_mu=mu, popart_sigma=sigma)

    args = [t[k] for k in ppof.INPUTS]
    eager = call(*[x.clone() if x is not None else None for x in args])
    torch._dynamo.reset()
    got = torch.compile(call, fullgraph=True)(*[x.clone() if x is not None else None for x in args])
    for k in ('adv', 'value', 'return_', 'return_stats', 'adv_stats'):
        a, b = getattr(got, k), getattr(eager, k)
        assert (a is None) == (b is None), k
        if a is not None:
            assert np.array_equal(_bits(a.cpu().numpy()), _bits(b.cpu().numpy())), k
    if case['mode'] in ('symlog', 'value_rescale'):  # as tests/test_ppof.py without the reference at hand
        scale = float(np.nanmax(np.abs(d['out_adv'][np.isfinite(d['out_adv'])])))
        for k, what in (('out_adv', 'adv'), ('out_value', 'value'), ('out_return', 'return_')):
            ppof.close(getattr(got, what).cpu().numpy(), d[k], 1e-5, scale, what)
    else:
        for k, what in (('out_adv', 'adv'), ('out_value', 'value'), ('out_return', 'return_')):
            ppof.same_bits(getattr(got, what).cpu().numpy(), d[k], what)


# ---------------------------------------------------------------------------------------------------------------------
# learner steps, model included
# ---------------------------------------------------------------------------------------------------------------------
def _sac_critic_step():
    """discrete-free SAC's twin critic (ding/policy/sac.py): two Q heads on (obs, action), one v_1step_td_error each"""
    torch.manual_seed(0)
    q1, q2 = (torch.nn.Sequential(torch.nn.Linear(8 + 2, 64), torch.nn.ReLU(), torch.nn.Linear(64, 1)).cuda()
              for _ in range(2))
    obs, act = torch.randn(256, 8, device='cuda'), torch.randn(256, 2, device='cuda')
    target_v, reward = torch.randn(256, device='cuda'), torch.randn(256, device='cuda')
    done = (torch.rand(256, device='cuda') < 0.1).float()

    def step(obs, act, target_v, reward, done):
        x = torch.cat([obs, act], dim=1)
        losses = []
        for q in (q1, q2):
            loss, td = api.v_1step_td_error(api.v_1step_td_data(q(x).squeeze(-1), target_v, reward, done, None), 0.99)
            losses.append(loss)
        return losses[0] + losses[1]
    return step, (obs, act, target_v, reward, done), list(q1.parameters()) + list(q2.parameters())


def _qrdqn_step():
    torch.manual_seed(1)
    A, n = 6, 32
    net = torch.nn.Sequential(torch.nn.Linear(16, 64), torch.nn.ReLU(), torch.nn.Linear(64, A * n)).cuda()
    obs, nobs = torch.randn(64, 16, device='cuda'), torch.randn(64, 16, device='cuda')
    act = torch.randint(0, A, (64, ), device='cuda')
    reward, done = torch.randn(3, 64, device='cuda'), (torch.rand(64, device='cuda') < 0.1).float()
    tau = ((torch.arange(n, device='cuda', dtype=torch.float32) + 0.5) / n).view(1, n, 1).expand(64, n, 1)

    def step(obs, nobs, act, reward, done):
        q = net(obs).view(64, A, n)
        with torch.no_grad():
            nq = net(nobs).view(64, A, n)
            nact = nq.mean(-1).argmax(-1)
        loss, td = api.qrdqn_nstep_td_error(api.qrdqn_nstep_td_data(q, nq, act, nact, reward, done, tau, None), 0.99,
                                            nstep=3)
        return loss, td.detach()
    return step, (obs, nobs, act, reward, done), list(net.parameters())


def _ppof_step():
    """PPOF's continuous learner step (ding/policy/ppof.py): the value-normalised advantage recompute under no_grad, then
    the policy loss on a Gaussian head"""
    torch.manual_seed(2)
    n, d = 128, 3
    actor = torch.nn.Linear(10, 2 * d).cuda()
    critic = torch.nn.Linear(10, 1).cuda()
    obs, nobs = torch.randn(n, 10, device='cuda'), torch.randn(n, 10, device='cuda')
    reward, done = torch.randn(n, device='cuda'), (torch.rand(n, device='cuda') < 0.05).float()
    act = torch.randn(n, d, device='cuda')
    mu_old, sigma_old = torch.randn(n, d, device='cuda'), torch.rand(n, d, device='cuda') + 0.5

    def step(obs, nobs, reward, done, act, mu_old, sigma_old):
        with torch.no_grad():
            v, nv = critic(obs).squeeze(-1), critic(nobs).squeeze(-1)
            ret = api.ppof_gae_returns(api.gae_data(v, nv, reward, done, done), 0.99, 0.95, value_norm='symlog')
        out = actor(obs)
        mu, sigma = out[:, :d], torch.nn.functional.softplus(out[:, d:]) + 1e-3
        adv = (ret.adv - ret.adv_stats[0]) / ret.adv_stats[1]
        loss, info = api.ppo_policy_error_continuous(api.ppo_policy_data_continuous(
            {'mu': mu, 'sigma': sigma}, {'mu': mu_old, 'sigma': sigma_old}, act, adv, None, None), 0.2)
        value_loss = ((critic(obs).squeeze(-1) - ret.return_) ** 2).mean()
        return loss.policy_loss - 0.01 * loss.entropy_loss + 0.5 * value_loss, info.approx_kl
    return step, (obs, nobs, reward, done, act, mu_old, sigma_old), list(actor.parameters()) + list(critic.parameters())


@pytest.mark.gpu
@pytest.mark.parametrize('make', (_sac_critic_step, _qrdqn_step, _ppof_step), ids=('sac_twin_critic', 'qrdqn', 'ppof'))
def test_learner_step_compiles_without_a_graph_break(make, monkeypatch):
    """the step's forward (model + loss) compiles as one graph; its backward runs the compiled backward graph"""
    monkeypatch.setattr(api.ppo, 'LAZY_INFO', True)
    step, args, params = make()
    torch._dynamo.reset()
    explain = torch._dynamo.explain(step)(*args)
    assert explain.graph_break_count == 0, [str(b.reason) for b in explain.break_reasons]

    def run(f):
        for p in params:
            p.grad = None
        out = f(*args)
        out[0].backward() if isinstance(out, tuple) else out.backward()
        return [x.detach().clone() for x in torch.utils._pytree.tree_leaves(out)], [p.grad.clone() for p in params]

    with _same_record() as restore:
        want, want_grads = run(step)
        restore()
        torch._dynamo.reset()
        got, got_grads = run(torch.compile(step, fullgraph=True))
    for a, b in zip(got, want):
        assert torch.allclose(a, b, rtol=1e-5, atol=1e-6), (a, b)
    for a, b in zip(got_grads, want_grads):
        assert torch.allclose(a, b, rtol=1e-4, atol=1e-6)
