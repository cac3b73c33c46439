"""torch.compile over the eight operators of the reference's plugin boundary (gae, ppo_error, q_nstep_td_error,
q_nstep_td_error_with_rescale, dist_nstep_td_error, td_lambda_error, upgo_loss, vtrace_error_discrete_action).

CPU part: against the logging stand-in for the CUDA library of ``tests/test_launch_log.py``, each loss compiles with
``fullgraph=True`` (no graph break) and its compiled forward + backward makes the same C-ABI calls, in the same order and
with the same int and float arguments, as the eager call on the same inputs.

GPU part: ``torch.library.opcheck`` on every ``b200rl`` op; inductor results bit-identical to eager on the edge cases of the
fp64 suites and within the suite's tolerances of the reference; a changing loss mix; ``mode="reduce-overhead"`` replays;
a dynamic batch dimension without recompiling.
"""
import contextlib

import numpy as np
import pytest
import torch
import torch._dynamo

import di_engine_b200 as b2
from di_engine_b200 import _lib, ops, torch_ops
from tests import cases
from tests.test_launch_log import _LoggingLib

api = b2.rl_utils
FUNCS = ('gae', 'ppo_error', 'q_nstep_td_error', 'q_nstep_td_error_with_rescale', 'dist_nstep_td_error', 'td_lambda_error',
         'upgo_loss', 'vtrace_error_discrete_action')
TD_FUNCS = ('q_nstep_td_error', 'q_nstep_td_error_with_rescale', 'dist_nstep_td_error')


@pytest.fixture(autouse=True)
def _distribution_validation():
    """dynamo turns off torch.distributions' argument validation for the whole process the first time it runs; the
    reference's errors that other tests check depend on it"""
    validate = torch.distributions.Distribution._validate_args
    yield
    torch.distributions.Distribution.set_default_validate_args(validate)


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the launch sequence of the compiled loss against the stand-in library
# ---------------------------------------------------------------------------------------------------------------------
@contextlib.contextmanager
def _stand_in():
    lib = _LoggingLib(1)
    keep = []
    data_ptr = torch.Tensor.data_ptr

    def keep_alive(t):
        keep.append(t)
        return data_ptr(t)

    def check(rc, what):
        assert rc == 0 and lib.log[-1]['check'] is None, (rc, what)
        lib.log[-1]['check'] = what

    ws = torch.zeros(1 << 18)
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(ops, 'lib', lambda: lib)
        mp.setattr(ops, 'require_cuda', lambda: None)
        mp.setattr(ops, 'compute_device', lambda *t: torch.device('cpu'))
        mp.setattr(ops, 'stream_ptr', lambda: 0)
        mp.setattr(ops, 'workspace', lambda dev: ws)
        mp.setattr(torch.cuda, 'device', lambda d: contextlib.nullcontext())
        mp.setattr(api.td, 'CHECK_DIST_POSITIVE', False)
        mp.setattr(api.ppo, 'LAZY_INFO', False)
        mp.setattr(_lib, 'check', check)
        mp.setattr(torch.Tensor, 'data_ptr', keep_alive)
        yield lib.log


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _rg(t):
    return t.requires_grad_(True)


B, N, T, NSTEP = 4, 5, 3, 3


def _ppo_in(g):
    return (api.ppo_data(_rg(torch.randn(B, N, generator=g)), torch.randn(B, N, generator=g),
                         torch.randint(0, N, (B, ), generator=g), _rg(torch.randn(B, generator=g)),
                         *(torch.randn(B, generator=g) for _ in range(3)), None, None), )


def _q_in(g):
    data = api.q_nstep_td_data(_rg(torch.randn(B, N, generator=g)), torch.randn(B, N, generator=g),
                               torch.randint(0, N, (B, ), generator=g), torch.randint(0, N, (B, ), generator=g),
                               torch.randn(NSTEP, B, generator=g), (torch.rand(B, generator=g) < 0.3).float(), None)
    return data, 0.95, NSTEP


def _dist_in(g):
    data = api.dist_nstep_td_data(_rg(torch.rand(B, N, 11, generator=g) + 0.1), torch.rand(B, N, 11, generator=g) + 0.1,
                                  torch.randint(0, N, (B, ), generator=g), torch.randint(0, N, (B, ), generator=g),
                                  torch.randn(NSTEP, B, generator=g), (torch.rand(B, generator=g) < 0.3).float(), None)
    return data, 0.95, -10.0, 10.0, 11, NSTEP


def _gae_in(g):
    return (api.gae_data(torch.randn(T, B, generator=g), torch.randn(T, B, generator=g), torch.randn(T, B, generator=g),
                         (torch.rand(T, B, generator=g) < 0.3).float(), None), 0.99, 0.95)


def _tdl_in(g):
    return (api.td_lambda_data(_rg(torch.randn(T + 1, B, generator=g)), torch.randn(T, B, generator=g), None), )


def _upgo_in(g):
    return (_rg(torch.randn(T, B, N, generator=g)), torch.rand(T, B, generator=g) + 0.5,
            torch.randint(0, N, (T, B), generator=g), torch.randn(T, B, generator=g), torch.randn(T + 1, B, generator=g))


def _vtrace_in(g):
    return (api.vtrace_data(_rg(torch.randn(T, B, N, generator=g)), torch.randn(T, B, N, generator=g),
                            torch.randint(0, N, (T, B), generator=g), _rg(torch.randn(T + 1, B, generator=g)),
                            torch.randn(T, B, generator=g), None), )


# name -> (inputs, the scalar to back-propagate from the function's result; None: no backward)
LOSSES = {
    'gae': (_gae_in, None),
    'ppo_error': (_ppo_in, lambda r: r[0].policy_loss + 0.5 * r[0].value_loss - 0.01 * r[0].entropy_loss),
    'q_nstep_td_error': (_q_in, lambda r: r[0]),
    'q_nstep_td_error_with_rescale': (_q_in, lambda r: r[0]),
    'dist_nstep_td_error': (_dist_in, lambda r: r[0]),
    'td_lambda_error': (_tdl_in, lambda r: r),
    'upgo_loss': (_upgo_in, lambda r: r),
    'vtrace_error_discrete_action': (_vtrace_in, lambda r: r.policy_loss + 0.5 * r.value_loss - 0.01 * r.entropy_loss),
}


def _launches(log):
    """the launches of a log: entry point, the name its check reports, and every argument -- a pointer only as whether it
    is null, which tells a verify launch (handed the forward's g_used and record) from a recompute (handed null)"""
    return [(e['fn'], e['check'], [(a is None) if ty is _lib.P else a for a, ty in zip(e['args'], _lib.PROTOTYPES[e['fn']])])
            for e in log if not e['fn'].endswith('_supported')]


def _queries(log):
    return [(e['fn'], [a is None for a in e['args']]) for e in log if e['fn'].endswith('_supported')]


def _td_per_sample_detached(fn):
    """``fn`` returning td_error_per_sample detached, as a learner takes it for priorities: an output of a compiled graph
    that the backward does not reach gets a zero gradient, which would make the backward recompute"""
    return lambda *a, **k: (lambda loss, per: (loss, per.detach()))(*fn(*a, **k))


def _step(fn, name):
    inputs, loss = LOSSES[name]
    args = inputs(_g(7))
    with _stand_in() as log:
        out = fn(*args)
        if loss is not None:
            loss(out).backward()
    return log


@pytest.mark.filterwarnings('ignore:invalid value encountered in cast')  # the stand-in leaves outputs uninitialised
@pytest.mark.parametrize('name', FUNCS)
def test_compiled_launch_sequence_matches_eager(name):
    fn = getattr(api, name)
    torch._dynamo.reset()
    want = _step(fn, name)
    if name in TD_FUNCS:
        fn = _td_per_sample_detached(fn)
    got = _step(torch.compile(fn, backend='aot_eager', fullgraph=True), name)
    assert len(want) > 0
    assert _launches(got) == _launches(want)
    # a custom op keeps no state between forward and backward: the backward op repeats the forward's question to the
    # library (the *_supported query, a host-side check of the buffers) to learn whether the forward wrote the gradients
    assert _queries(got) == _queries(want) * (2 if _queries(want) else 1)


@pytest.mark.filterwarnings('ignore:invalid value encountered in cast')
def test_graph_breaking_function_with_scalar_value_gamma_runs_compiled():
    """a function outside the eight keeps its autograd.Function: dynamo breaks the graph there and runs it eagerly, with
    the scalar value_gamma it was given (read from the cached device constant, as without torch.compile)"""
    from tests.test_launch_log import _q_inputs

    def qrdqn():
        q, nq, act, nact, reward, done = _q_inputs(_g(9), (B, N, 3))
        loss, _ = api.qrdqn_nstep_td_error(api.qrdqn_nstep_td_data(q, nq, act, nact, reward, done, 3, None), 0.95,
                                           nstep=NSTEP, value_gamma=0.9)
        loss.backward()

    def compiled():
        q, nq, act, nact, reward, done = _q_inputs(_g(9), (B, N, 3))
        f = torch.compile(lambda *a, **k: api.qrdqn_nstep_td_error(*a, **k)[0], backend='aot_eager')
        f(api.qrdqn_nstep_td_data(q, nq, act, nact, reward, done, 3, None), 0.95, nstep=NSTEP, value_gamma=0.9).backward()

    torch._dynamo.reset()
    with _stand_in() as want:
        qrdqn()
    with _stand_in() as got:
        compiled()
    assert [e['fn'] for e in want] == ['b200rl_quantile_td_fwd', 'b200rl_quantile_td_bwd']
    assert _launches(got) == _launches(want)


def test_gae_masks_next_value_in_place_when_compiled():
    args = _gae_in(_g(5))
    torch._dynamo.reset()
    with _stand_in() as log:
        torch.compile(api.gae, backend='aot_eager', fullgraph=True)(*args)
    assert [e['fn'] for e in log] == ['b200rl_gae']
    schema = torch.ops.b200rl.gae.default._schema
    assert [a.name for a in schema.arguments if a.alias_info is not None and a.alias_info.is_write] == ['next_value']


def test_ops_schemas_hold_only_tensors_and_scalars():
    for name in ('gae', 'ppo_loss', 'ppo_bwd', 'qntd_fwd', 'qntd_bwd', 'dntd_fwd', 'dntd_bwd', 'td_lambda_fwd', 'scale',
                 'lambda_returns', 'upgo_fwd', 'upgo_bwd', 'vtrace_loss', 'vtrace_bwd'):
        schema = getattr(torch.ops.b200rl, name).default._schema
        for a in schema.arguments:
            assert str(a.type) in ('Tensor', 'Optional[Tensor]', 'SymInt', 'int', 'float', 'Optional[float]', 'bool', 'str'), (
                name, a.name, a.type)


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
class _CompiledAPI:
    """The reference's names, with the eight functions compiled; td_error_per_sample leaves the graph detached (as a
    learner uses it, for priorities), so the backward of the loss alone keeps the forward-written gradient.  ppo_error's
    graph keeps its two monitors on the device (``LAZY_INFO``): the python floats of ``.item()`` leave an inductor graph
    through a CPU kernel, which needs a host C++ toolchain with OpenMP; they are read after the call instead."""

    def __init__(self, **kw):
        for name in FUNCS:
            fn = getattr(api, name)
            if name in TD_FUNCS:
                fn = _td_per_sample_detached(fn)
            setattr(self, name, torch.compile(fn, fullgraph=True, **kw))
        compiled_ppo = self.ppo_error

        def ppo_error(*a, **k):
            lazy, api.ppo.LAZY_INFO = api.ppo.LAZY_INFO, True
            try:
                loss, info = compiled_ppo(*a, **k)
            finally:
                api.ppo.LAZY_INFO = lazy
            return loss, api.ppo_info(*(float(x) for x in info))

        self.ppo_error = ppo_error

    def __getattr__(self, name):
        return getattr(api, name)


@contextlib.contextmanager
def _same_record():
    """Let the enclosed code run twice from the same upstream-gradient records: a backward launch refreshes the record when
    the upstream gradients differ from it, and which of its two branches runs (verify, or recompute) decides the last bits
    of the gradients.  Yields a callable that puts the records back as they were on entry."""
    saved = {k: h.clone() for k, h in ops._HINT.items()}

    def restore():
        for (dev, kind), h in ops._HINT.items():
            h.copy_(saved[(dev, kind)] if (dev, kind) in saved else torch.tensor(ops._HINT_INIT[kind]))

    yield restore


# the edge cases of the fp64 suites for the eight functions
GPU_CASES = ('gae_T1', 'gae_1d', 'gae_marl', 'gae_bool', 'ppo_marl', 'ppo_marl_dc', 'ppo_kl_k3', 'ppo_wideN', 'ppo_one',
             'qntd_cum', 'qntd_cfgB', 'qntd_vg_float', 'qntd_ngu', 'qntd_marl_branch', 'qntdr_n5_w_vg', 'dntd_cfgC',
             'dntd_w_float', 'dntd_marl', 'tdl_T1', 'tdl_w', 'upgo_3d_big', 'upgo_4d_mask', 'vtrace_cfgE', 'vtrace_clips',
             'vtrace_done_heavy')


def _gpu_cases():
    c = cases.build_cases()
    # a done-heavy V-trace batch: IMPALA's masking of value / reward / weight at the episode ends of half the steps
    op, t, p = cases.vtrace_case(83, 24, 16, 6, weight='tensor', gamma=0.99, lambda_=0.95)
    done = (torch.rand(24, 16, generator=torch.Generator().manual_seed(84)) < 0.5).float()
    t['value'], t['reward'], t['weight'] = (x.detach() for x in api.impala_reshape_data(t['value'], t['reward'], done))
    c['vtrace_done_heavy'] = (op, t, p)
    return c


@pytest.fixture
def compiled():
    torch._dynamo.reset()
    return _CompiledAPI()


@pytest.mark.gpu
@pytest.mark.parametrize('name', GPU_CASES)
def test_inductor_bit_identical_to_eager_and_within_reference_tolerance(name, compiled):
    from oracle import rl_oracle
    op, t, p = _gpu_cases()[name]
    with _same_record() as restore:
        want = cases.run_api(api, op, t, p, device='cuda:0')
        restore()
        got = cases.run_api(compiled, op, t, p, device='cuda:0')
    cases.compare(got, want, exact=True)
    ref = cases.run_oracle(rl_oracle, op, t, p)
    if op == 'gae':
        cases.compare(got, ref, exact=True)
    else:
        cases.compare(got, ref, rtol=1e-5, atol=1e-5)


def _recording():
    """every b200rl op call of the enclosed code: (op, args, kwargs)"""
    from torch.utils._python_dispatch import TorchDispatchMode
    calls = []

    class Record(TorchDispatchMode):

        def __torch_dispatch__(self, func, types, args=(), kwargs=None):
            if func.namespace == 'b200rl':
                calls.append((func, args, kwargs or {}))
            return func(*args, **(kwargs or {}))

    return Record(), calls


@pytest.mark.gpu
@pytest.mark.parametrize('name', FUNCS)
def test_opcheck(name):
    inputs, loss = LOSSES[name]
    args = [x.cuda() if isinstance(x, torch.Tensor) else x for x in inputs(_g(11))]
    args = [type(a)(*[x.detach().cuda().requires_grad_(x.requires_grad) if isinstance(x, torch.Tensor) else x for x in a])
            if isinstance(a, tuple) else a for a in args]
    if name == 'upgo_loss':
        args = [x.detach().cuda().requires_grad_(x.requires_grad) for x in inputs(_g(11))]
    mode, calls = _recording()
    fn = getattr(api, name)
    with mode, pytest.MonkeyPatch.context() as mp:
        mp.setattr(torch.compiler, 'is_compiling', lambda: True)  # the traced path, run eagerly
        mp.setattr(api.ppo, 'LAZY_INFO', True)
        out = fn(*args)
        if loss is not None:
            loss(out).backward()
    seen = set()
    for op, a, k in calls:
        if op in seen:
            continue
        seen.add(op)
        if op._opname.endswith('_bwd') or op._opname == 'scale':  # a backward op is not differentiated again
            a, k = torch.utils._pytree.tree_map_only(torch.Tensor, lambda x: x.detach(), (a, k))
        # the forward-written gradients are those of the upstream-gradient record, which opcheck's own backward passes
        # refresh: each call gets the initial record, so that its outputs are a function of its inputs
        with pytest.MonkeyPatch.context() as mp:
            mp.setattr(ops, 'ppo_hint', lambda dev, kind='ppo': torch.tensor(ops._HINT_INIT[kind], device=dev))
            torch.library.opcheck(op, a, k)
    assert seen


def _ppo_tensors(seed, S, n=6, dev='cuda:0'):
    g = _g(seed)
    return [torch.randn(S, n, generator=g).to(dev).requires_grad_(True), torch.randn(S, n, generator=g).to(dev),
            torch.randint(0, n, (S, ), generator=g).to(dev), torch.randn(S, generator=g).to(dev).requires_grad_(True)] + \
        [torch.randn(S, generator=g).to(dev) for _ in range(3)]


def _ppo_step(fn, ts, mix):
    loss, info = fn(api.ppo_data(*ts, None, None))
    total = mix[0] * loss.policy_loss + mix[1] * loss.value_loss + mix[2] * loss.entropy_loss
    ln, vn = ts[0], ts[3]
    gl, gv = torch.autograd.grad(total, (ln, vn))
    return [x.detach().clone() for x in (loss.policy_loss, loss.value_loss, loss.entropy_loss, gl, gv) + tuple(info)]


@pytest.mark.gpu
def test_changing_loss_mix_stays_exact_when_compiled(monkeypatch):
    monkeypatch.setattr(api.ppo, 'LAZY_INFO', True)
    torch._dynamo.reset()
    fn = torch.compile(api.ppo_error, fullgraph=True)
    for i, mix in enumerate(([1.0, 0.25, -0.01], [1.0, 1.0, -0.01], [1.0, 0.25, -0.01], [0.5, 1.0, 0.0])):
        ts = _ppo_tensors(20 + i, 64)
        with _same_record() as restore:
            want = _ppo_step(api.ppo_error, ts, mix)
            restore()
            got = _ppo_step(fn, ts, mix)
        for a, b in zip(got, want):
            assert np.array_equal(np.asarray(a.cpu() if isinstance(a, torch.Tensor) else a),
                                  np.asarray(b.cpu() if isinstance(b, torch.Tensor) else b)), mix


def _pool_of(t):
    """the memory pool id of the segment holding ``t``: (0, 0) is the ordinary pool, anything else a CUDA graph's"""
    for seg in torch.cuda.memory_snapshot():
        if seg['address'] <= t.data_ptr() < seg['address'] + seg['total_size']:
            return tuple(seg['segment_pool_id'])
    raise AssertionError('no segment holds the tensor')


@pytest.mark.gpu
@pytest.mark.parametrize('name', ('ppo_error', 'q_nstep_td_error', 'dist_nstep_td_error', 'vtrace_error_discrete_action',
                                  'gae'))
def test_reduce_overhead_replays_bit_identical_to_eager(name, monkeypatch):
    monkeypatch.setattr(api.ppo, 'LAZY_INFO', True)  # a graph that reads the device on the host is not replayed
    monkeypatch.setattr(api.td, 'CHECK_DIST_POSITIVE', False)  # a host read as well
    # no workspace, record or constant exists yet: the compiled call's warm-up is the first to need them
    lasting_buffers = {'_WS': {}, '_HINT': {}, '_CONST': {}}
    for k, v in lasting_buffers.items():
        monkeypatch.setattr(ops, k, v)
    monkeypatch.setattr(api.td, '_SUPPORT_CACHE', {})
    inputs, loss = LOSSES[name]
    kw = {'value_gamma': 0.9} if name == 'dist_nstep_td_error' else {}  # a python scalar: a cached device constant
    f = getattr(api, name)
    torch._dynamo.reset()
    fn = torch.compile(_td_per_sample_detached(f) if name in TD_FUNCS else f, mode='reduce-overhead', fullgraph=True)

    def to_cuda(x):
        if isinstance(x, torch.Tensor):
            return x.detach().cuda().requires_grad_(x.requires_grad)
        if isinstance(x, tuple) and hasattr(x, '_fields'):
            return type(x)(*[to_cuda(y) for y in x])
        return x

    def run(f, args):
        out = f(*args, **kw)
        flat = [x for x in torch.utils._pytree.tree_leaves(out) if isinstance(x, torch.Tensor)]
        res = [x.detach().clone() for x in flat]
        if loss is not None:
            leaves = [x for x in torch.utils._pytree.tree_leaves(args) if isinstance(x, torch.Tensor) and x.requires_grad]
            res += [g.clone() for g in torch.autograd.grad(loss(out), leaves)]
        else:
            res += [args[0].next_value.clone()]
        return res

    allocated = []
    lasting = ops.lasting
    monkeypatch.setattr(ops, 'lasting', lambda make, dev: allocated.append(dev) or lasting(make, dev))
    for step in range(22):  # 2 warm-up / record calls, then 20 replays
        args = [to_cuda(x) for x in inputs(_g(100 + step))]
        with _same_record() as restore:
            got = run(fn, args)
            restore()
            want = run(f, [to_cuda(x) for x in inputs(_g(100 + step))])
        for a, b in zip(got, want):
            assert torch.equal(a, b), (name, step)
        if step == 1:
            allocated.clear()
    assert allocated == [], 'a workspace or record was allocated after warm-up'
    buffers = [t for d in lasting_buffers.values() for t in d.values()] + list(api.td._SUPPORT_CACHE.values())
    if name != 'gae':  # the 2-D gae kernel takes no workspace
        assert len(lasting_buffers['_WS']) >= 2  # the graphs' stream and the eager one
    if name in ('ppo_error', 'vtrace_error_discrete_action'):
        assert lasting_buffers['_HINT']
    if name == 'dist_nstep_td_error':
        assert lasting_buffers['_CONST'] and api.td._SUPPORT_CACHE
    assert [_pool_of(t) for t in buffers] == [(0, 0)] * len(buffers)


@pytest.mark.gpu
def test_workspace_first_needed_inside_a_capture_raises():
    dev = torch.device('cuda:0')
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with pytest.raises(_lib.B200RLError, match='warm-up'):
        with torch.cuda.graph(g, stream=s):
            ops.lasting(lambda: torch.zeros(4, device=dev), dev)


@pytest.mark.gpu
@pytest.mark.parametrize('name', ('ppo_error', 'q_nstep_td_error'))
def test_dynamic_batch_does_not_recompile(name, monkeypatch):
    from torch._dynamo.utils import counters
    monkeypatch.setattr(api.ppo, 'LAZY_INFO', True)
    torch._dynamo.reset()
    counters.clear()
    fn = torch.compile(getattr(api, name), fullgraph=True)

    def args(S, seed):
        g = _g(seed)
        if name == 'ppo_error':
            ts = _ppo_tensors(seed, S)
            for t in ts:
                torch._dynamo.mark_dynamic(t, 0)
            return (api.ppo_data(*ts, None, None), )
        ts = [torch.randn(S, 6, generator=g), torch.randn(S, 6, generator=g), torch.randint(0, 6, (S, ), generator=g),
              torch.randint(0, 6, (S, ), generator=g), torch.randn(3, S, generator=g),
              (torch.rand(S, generator=g) < 0.2).float()]
        ts = [t.cuda() for t in ts]
        ts[0].requires_grad_(True)
        for i, t in enumerate(ts):
            torch._dynamo.mark_dynamic(t, 1 if i == 4 else 0)
        return api.q_nstep_td_data(*ts, None), 0.95, 3

    for S in (64, 320):
        a = args(S, S)
        want = getattr(api, name)(*a)
        got = fn(*a)
        assert torch.equal(got[0] if name != 'ppo_error' else got[0].policy_loss,
                           want[0] if name != 'ppo_error' else want[0].policy_loss)
    assert counters['stats']['unique_graphs'] == 1, dict(counters['stats'])
