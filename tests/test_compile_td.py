"""torch.compile over the value-based losses that ran on ``autograd.Function``s and so broke the graph: the DQfD losses
(``dqfd_nstep_td_error``, ``dqfd_nstep_td_error_with_rescale`` and R2D3's ``dqfd_nstep_td_error_sequence``), the soft TD
losses (``m_q_1step_td_error``, ``q_nstep_sql_td_error``, ``q_v_1step_td_error``), the R2D2 / NGU loop
``q_nstep_td_error_sequence`` and FQF's ``fqf_calculate_fraction_loss``.

CPU part: against the logging stand-in for the CUDA library of ``tests/test_launch_log.py``, each function compiles with
``backend='aot_eager', fullgraph=True`` and its compiled forward + backward makes exactly the launches of the eager call;
the ``*_supported`` queries are unchanged; every error the eager call raises on bad input is raised while compiling; every
new op schema holds tensors and scalars only; and every function of ``TRACED`` has a case.

GPU part: ``torch.library.opcheck`` on every new op; inductor results bit-identical to eager and within the suites'
tolerances of the stored reference values on the golden sets ``tests/golden/{dqfd,soft_td,fqf_fraction}``;
``mode="reduce-overhead"`` replays; a dynamic batch without recompiling; five learner steps, model included, that compile
without a graph break.
"""
import math

import numpy as np
import pytest
import torch
import torch._dynamo
import torch.nn as nn

import di_engine_b200 as b2
from di_engine_b200 import ops
from tests import test_dqfd as dqfd_suite, test_fqf_fraction as fraction_suite, test_soft_td as soft_suite
from tests.test_compile import _launches, _queries, _same_record, _stand_in
from tests.test_compile_all import _cuda, _recording
from tests.test_launch_log import _q_inputs

api = b2.rl_utils
B, N, NSTEP, T = 4, 5, 3, 3

# the public functions this file compiles
TRACED = ('dqfd_nstep_td_error', 'dqfd_nstep_td_error_with_rescale', 'dqfd_nstep_td_error_sequence',
          'q_nstep_td_error_sequence', 'm_q_1step_td_error', 'q_nstep_sql_td_error', 'q_v_1step_td_error',
          'fqf_calculate_fraction_loss')
NEW_OPS = ('qntd_seq_fwd', 'qntd_seq_bwd', 'dqfd_fwd', 'dqfd_bwd', 'soft_td_fwd', 'fqf_fraction_fwd', 'fqf_fraction_bwd')


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


class _LogCosh(nn.Module):
    """a criterion the kernels do not know: it runs as torch ops around the kernel's detached targets"""

    def forward(self, a, b):
        return torch.log(torch.cosh(a - b))


def _h(x):  # value rescaling, but not the library's own functions: the custom-transform path
    return torch.sign(x) * (torch.sqrt(torch.abs(x) + 1) - 1) + 0.01 * x


def _h_inv(x):
    return api.value_inv_transform(x)


# ---------------------------------------------------------------------------------------------------------------------
# the cases: name -> (inputs(g) -> args, fn(*args) -> the differentiable outputs to back-propagate)
# ---------------------------------------------------------------------------------------------------------------------
def _dqfd_in(cum=False, expert='float', rows=None):
    def inputs(g):
        shape = (B, N) if rows is None else (rows, B, N)
        lead = (B, ) if rows is None else (rows, B)
        q, nq = _rg(torch.randn(*shape, generator=g)), torch.randn(*shape, generator=g)
        act, nact, nact1 = (torch.randint(0, N, lead, generator=g) for _ in range(3))
        nq1 = torch.randn(*shape, generator=g)
        if rows is not None:
            reward = torch.randn(rows, NSTEP, B, generator=g)
        else:
            reward = torch.randn(B, generator=g) if cum else torch.randn(NSTEP, B, generator=g)
        done, done1 = ((torch.rand(*lead, generator=g) < 0.3).float() for _ in range(2))
        weight = torch.rand(*lead, generator=g)
        ie = {'float': (torch.rand(*lead, generator=g) < 0.5).float(), 'bool': torch.rand(*lead, generator=g) < 0.5,
              'scalar': 1.0}[expert]
        return api.dqfd_nstep_td_data(q, nq, act, nact, reward, done, done1, weight, nq1, nact1, ie),
    return inputs


def _dqfd_fn(name='dqfd_nstep_td_error', every_output=False, **kw):
    fn = getattr(api, name)

    def call(data):
        if name == 'dqfd_nstep_td_error_with_rescale':
            loss, per, stats = fn(data, 0.97, 1.0, 1.0, 0.6, 0.8, nstep=NSTEP, **kw)
        else:
            loss, per, stats = fn(data, 0.97, 1.0, 1.0, 0.8, 0.6, nstep=NSTEP, **kw)
        # a learner back-propagates the loss and detaches the per-sample error (priorities) and the statistics
        return (loss, per) + tuple(stats) if every_output else (loss, )
    return call


def _dqfd_seq_fn(**kw):
    def call(data):
        loss, prio, per, stats = api.dqfd_nstep_td_error_sequence(data, 0.97, 1.0, 1.0, 0.8, 0.6, nstep=NSTEP, **kw)
        return (loss, )
    return call


def _seq_in(ngu=False):
    def inputs(g):
        q, nq = _rg(torch.randn(T, B, N, generator=g)), torch.randn(T, B, N, generator=g)
        act, nact = torch.randint(0, N, (T, B), generator=g), torch.randint(0, N, (T, B), generator=g)
        reward, done = torch.randn(T, NSTEP, B, generator=g), (torch.rand(T, B, generator=g) < 0.3).float()
        weight = torch.rand(T, B, generator=g)
        gamma = [torch.tensor(0.9 + 0.02 * i) for i in range(B)] if ngu else 0.97
        return api.q_nstep_td_seq_data(q, nq, act, nact, reward, done, weight), gamma
    return inputs


def _seq_fn(**kw):
    def call(data, gamma):
        loss, prio, per = api.q_nstep_td_error_sequence(data, gamma, nstep=NSTEP, **kw)
        return (loss, )
    return call


def _mq_in(g):
    q, nq, act, _, reward, done = _q_inputs(g, (B, N))
    return api.m_q_1step_td_data(q, torch.randn(B, N, generator=g), nq, act, reward[0], done, torch.rand(B, generator=g)),


def _sql_in(cum=False):
    def inputs(g):
        q, nq, act, nact, reward, done = _q_inputs(g, (B, N))
        return api.q_nstep_td_data(q, nq, act, nact, reward[0] if cum else reward, done, None),
    return inputs


def _qv_in(g):
    q, _, act, _, reward, done = _q_inputs(g, (B, N))
    return api.q_v_1step_td_data(q, torch.randn(B, generator=g), act, reward[0], done, None),


def _fraction_in(g):
    """every operand a transposed view: (B, A, n) and (n, B) storage read as (B, n, A) and (B, n)"""
    A = 3
    q_tau_i = torch.randn(B, A, N - 1, generator=g).transpose(1, 2)
    q_value = _rg(torch.randn(B, A, N, generator=g)).transpose(1, 2)
    p = torch.softmax(torch.randn(B, N, generator=g), 1)
    quantiles = _rg(torch.cat([torch.zeros(B, 1), p.cumsum(1)], 1).t().contiguous()).t()
    return q_tau_i, q_value, quantiles, torch.randint(0, A, (B, ), generator=g)


CASES = {
    'dqfd_nstep_td_error': (_dqfd_in(), _dqfd_fn()),
    'dqfd_nstep_td_error[cum_reward]': (_dqfd_in(cum=True), _dqfd_fn(cum_reward=True)),
    'dqfd_nstep_td_error[value_gamma_scalar]': (_dqfd_in(), _dqfd_fn(value_gamma=0.9)),
    'dqfd_nstep_td_error[value_gamma_tensor]': (_dqfd_in(), _dqfd_fn(value_gamma=torch.linspace(0.8, 0.95, B))),
    'dqfd_nstep_td_error[is_expert_scalar]': (_dqfd_in(expert='scalar'), _dqfd_fn()),
    'dqfd_nstep_td_error[is_expert_bool]': (_dqfd_in(expert='bool'), _dqfd_fn()),
    'dqfd_nstep_td_error[criterion]': (_dqfd_in(), _dqfd_fn(criterion=_LogCosh())),
    'dqfd_nstep_td_error[every_output]': (_dqfd_in(), _dqfd_fn(every_output=True)),
    'dqfd_nstep_td_error_with_rescale': (_dqfd_in(), _dqfd_fn('dqfd_nstep_td_error_with_rescale')),
    'dqfd_nstep_td_error_with_rescale[custom_transform]': (
        _dqfd_in(), _dqfd_fn('dqfd_nstep_td_error_with_rescale', trans_fn=_h, inv_trans_fn=_h_inv)),
    'dqfd_nstep_td_error_sequence': (_dqfd_in(rows=T), _dqfd_seq_fn(value_gamma=torch.full((T, B), 0.9))),
    'dqfd_nstep_td_error_sequence[rescale]': (_dqfd_in(rows=T, expert='bool'), _dqfd_seq_fn(rescale=True)),
    'q_nstep_td_error_sequence': (_seq_in(), _seq_fn(value_gamma=torch.full((T, B), 0.9))),
    'q_nstep_td_error_sequence[rescale]': (_seq_in(), _seq_fn(rescale=True, priority_mix=0.7)),
    'q_nstep_td_error_sequence[ngu]': (_seq_in(ngu=True), _seq_fn(rescale=True)),
    'm_q_1step_td_error': (_mq_in, lambda data: api.m_q_1step_td_error(data, 0.99, 0.03, 0.9)[:1]),
    'm_q_1step_td_error[criterion]': (_mq_in, lambda data: api.m_q_1step_td_error(data, 0.99, 0.03, 0.9, _LogCosh())[:1]),
    'q_nstep_sql_td_error': (_sql_in(), lambda data: api.q_nstep_sql_td_error(data, 0.99, 0.1, nstep=NSTEP)[:1]),
    'q_nstep_sql_td_error[cum_reward]': (_sql_in(cum=True), lambda data: api.q_nstep_sql_td_error(
        data, 0.99, 0.1, nstep=NSTEP, cum_reward=True)[:1]),
    'q_nstep_sql_td_error[value_gamma]': (_sql_in(), lambda data: api.q_nstep_sql_td_error(
        data, 0.99, 0.1, nstep=NSTEP, value_gamma=torch.linspace(0.8, 0.95, B))[:1]),
    'q_nstep_sql_td_error[value_gamma_scalar]': (_sql_in(), lambda data: api.q_nstep_sql_td_error(
        data, 0.99, 0.1, nstep=NSTEP, value_gamma=0.9)[:1]),
    'q_v_1step_td_error': (_qv_in, lambda data: api.q_v_1step_td_error(data, 0.99)[:1]),
    'q_v_1step_td_error[every_output]': (_qv_in, lambda data: api.q_v_1step_td_error(data, 0.99)),
    'fqf_calculate_fraction_loss': (_fraction_in, lambda *a: (api.fqf_calculate_fraction_loss(*a), )),
}
MIX = (1.0, 0.5, -0.4, 0.7, 1.3)


def _run(fn, name, seed=7):
    inputs, _ = CASES[name]
    args = inputs(_g(seed))
    with _stand_in() as log:
        outs = fn(*args)
        sum(w * o for w, o in zip(MIX, outs)).sum().backward()
    return log


def test_every_traced_function_has_a_case():
    assert all(callable(getattr(api, name, None)) for name in TRACED)
    assert sorted(set(TRACED) - {name.split('[')[0] for name in CASES}) == []


@pytest.mark.filterwarnings('ignore:invalid value encountered in cast')  # the stand-in leaves outputs uninitialised
@pytest.mark.parametrize('name', sorted(CASES))
def test_compiled_launch_sequence_matches_eager(name):
    fn = CASES[name][1]
    torch._dynamo.reset()
    want = _run(fn, name)
    got = _run(torch.compile(fn, backend='aot_eager', fullgraph=True), name)
    assert len(want) > 0
    assert _launches(got) == _launches(want)
    assert _queries(got) == _queries(want)


def _bad_inputs():
    g = _g(3)
    dq = _dqfd_in()(g)[0]
    ds = _dqfd_in(rows=T)(g)[0]
    sq, sg = _seq_in()(g)
    mq = _mq_in(g)[0]
    qn = _sql_in()(g)[0]
    qv = _qv_in(g)[0]
    fr = _fraction_in(g)
    return {
        'dqfd_nstep_td_error[list_gamma]': (NotImplementedError, lambda: api.dqfd_nstep_td_error(
            dq, [0.9] * B, 1.0, 1.0, 0.8, nstep=NSTEP)),
        'dqfd_nstep_td_error[shape]': (ValueError, lambda: api.dqfd_nstep_td_error(
            dq._replace(next_n_q=dq.next_n_q[:2]), 0.97, 1.0, 1.0, 0.8, nstep=NSTEP)),
        'dqfd_nstep_td_error_with_rescale[is_expert]': (ValueError, lambda: api.dqfd_nstep_td_error_with_rescale(
            dq._replace(is_expert=dq.is_expert[:2]), 0.97, 1.0, 1.0, 1.0, 0.8, nstep=NSTEP)),
        'dqfd_nstep_td_error_sequence[shape]': (ValueError, lambda: api.dqfd_nstep_td_error_sequence(
            ds._replace(reward=ds.reward[:, :, :2]), 0.97, 1.0, 1.0, 0.8, nstep=NSTEP)),
        'dqfd_nstep_td_error_sequence[criterion]': (NotImplementedError, lambda: api.dqfd_nstep_td_error_sequence(
            ds, 0.97, 1.0, 1.0, 0.8, nstep=NSTEP, criterion=_LogCosh())),
        'q_nstep_td_error_sequence[shape]': (ValueError, lambda: api.q_nstep_td_error_sequence(
            sq._replace(done=sq.done[:, :2]), sg, nstep=NSTEP)),
        'q_nstep_td_error_sequence[criterion]': (NotImplementedError, lambda: api.q_nstep_td_error_sequence(
            sq, sg, nstep=NSTEP, criterion=_LogCosh())),
        'm_q_1step_td_error[bool_done]': (RuntimeError, lambda: api.m_q_1step_td_error(
            mq._replace(done=mq.done > 0), 0.99, 0.03, 0.9)),
        'm_q_1step_td_error[N<2]': (RuntimeError, lambda: api.m_q_1step_td_error(
            mq._replace(q=mq.q[:, :1], target_q=mq.target_q[:, :1], next_q=mq.next_q[:, :1], act=mq.act * 0),
            0.99, 0.03, 0.9)),
        'm_q_1step_td_error[shape]': (ValueError, lambda: api.m_q_1step_td_error(
            mq._replace(target_q=mq.target_q[:2]), 0.99, 0.03, 0.9)),
        'q_nstep_sql_td_error[list_gamma]': (NotImplementedError, lambda: api.q_nstep_sql_td_error(
            qn, [0.9] * B, 0.1, nstep=NSTEP)),
        'q_nstep_sql_td_error[bool_done]': (RuntimeError, lambda: api.q_nstep_sql_td_error(
            qn._replace(done=qn.done > 0), 0.99, 0.1, nstep=NSTEP)),
        'q_nstep_sql_td_error[shape]': (ValueError, lambda: api.q_nstep_sql_td_error(
            qn._replace(reward=qn.reward[:, :2]), 0.99, 0.1, nstep=NSTEP)),
        'q_v_1step_td_error[bool_done]': (RuntimeError, lambda: api.q_v_1step_td_error(
            qv._replace(done=qv.done > 0), 0.99)),
        'q_v_1step_td_error[shape]': (ValueError, lambda: api.q_v_1step_td_error(qv._replace(v=qv.v[:2]), 0.99)),
        'fqf_calculate_fraction_loss[requires_grad]': (AssertionError, lambda: api.fqf_calculate_fraction_loss(
            fr[0], fr[1].detach(), fr[2], fr[3])),
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
    # an assertion that dynamo meets while tracing keeps its message and gains dynamo's "from user code" trailer
    assert str(compiled.value).split('\n\nfrom user code:')[0] == str(eager.value)


def test_new_ops_schemas_hold_only_tensors_and_scalars():
    for name in NEW_OPS:
        schema = getattr(torch.ops.b200rl, name).default._schema
        for a in schema.arguments:
            assert str(a.type) in ('Tensor', 'Optional[Tensor]', 'SymInt', 'int', 'float', 'Optional[float]', 'bool', 'str'), (
                name, a.name, a.type)


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
OPCHECK_CASES = ('dqfd_nstep_td_error[value_gamma_scalar]', 'dqfd_nstep_td_error[is_expert_scalar]',
                 'dqfd_nstep_td_error[every_output]', 'dqfd_nstep_td_error_sequence', 'q_nstep_td_error_sequence[ngu]',
                 'm_q_1step_td_error', 'q_nstep_sql_td_error[value_gamma_scalar]', 'q_v_1step_td_error[every_output]',
                 'fqf_calculate_fraction_loss')


@pytest.mark.gpu
def test_opcheck():
    seen = set()
    for name in OPCHECK_CASES:
        inputs, fn = CASES[name]
        args = _on_cuda(inputs(_g(11)))
        mode, calls = _recording()
        with mode, pytest.MonkeyPatch.context() as mp:
            mp.setattr(torch.compiler, 'is_compiling', lambda: True)  # the traced path, run eagerly
            outs = fn(*args)
            sum(w * o for w, o in zip(MIX, outs)).sum().backward()
        for op, a, k in calls:
            if op in seen:
                continue
            seen.add(op)
            if op._opname.endswith('_bwd'):  # a backward op is not differentiated again
                a, k = torch.utils._pytree.tree_map_only(torch.Tensor, lambda x: x.detach(), (a, k))
            torch.library.opcheck(op, a, k)
    assert set(NEW_OPS) <= {op._opname for op in seen}


def _on_cuda(args):
    """``_cuda`` of every argument, the tensors of NGU's list gamma included"""
    return tuple([_cuda(x) for x in a] if isinstance(a, list) else _cuda(a) for a in args)


def _results(outs, args):
    """every tensor a call returned, then the gradients of its inputs that require grad (those the loss reaches: q_value
    of the fraction loss gets none)"""
    res = [o.detach().clone() for o in outs]
    leaves = [x for x in torch.utils._pytree.tree_leaves(args) if isinstance(x, torch.Tensor) and x.requires_grad]
    grads = torch.autograd.grad(sum(w * o for w, o in zip(MIX, outs)).sum(), leaves, allow_unused=True)
    return res + [g.clone() for g in grads if g is not None]


def _compiled(fn):
    torch._dynamo.reset()
    return torch.compile(fn, fullgraph=True)


class _CompiledAPI:
    """the reference's names, with the functions a golden-set suite calls compiled (inductor, fullgraph)"""

    def __init__(self, *names):
        for name in names:
            setattr(self, name, _compiled(getattr(api, name)))

    def __getattr__(self, name):
        return getattr(api, name)


def _same_bits(got, want):
    assert set(got) == set(want)
    for k in want:
        assert np.array_equal(np.asarray(got[k], np.float32), np.asarray(want[k], np.float32), equal_nan=True), k


def _torch_callables(case):
    """a case whose criterion or value transform is a torch callable: under inductor those run as inductor's own kernels,
    fused with the sums around them, which may round differently from eager torch in the last bit"""
    return case['crit'] == 'quartic' or case.get('custom_trans', False)


@pytest.mark.gpu
@pytest.mark.parametrize('name', dqfd_suite.fixture_names())
def test_dqfd_fixtures_compiled(name):
    """the DQfD golden set, every output back-propagated (tests/test_dqfd.py's mix): bit-identical to eager (within that
    suite's tolerance where the case runs a torch criterion or transform), and within that suite's tolerance of the stored reference
    outputs and gradients"""
    case, t, want = dqfd_suite.load_fixture(name)
    compiled = _CompiledAPI('dqfd_nstep_td_error', 'dqfd_nstep_td_error_with_rescale')
    eager = dqfd_suite.run(api, case, t, 'cuda')
    got = dqfd_suite.run(compiled, case, t, 'cuda')
    if _torch_callables(case):
        dqfd_suite.compare(got, eager)
    else:
        _same_bits(got, eager)
    dqfd_suite.compare(got, want)


@pytest.mark.gpu
@pytest.mark.filterwarnings('ignore:Using a target size')
@pytest.mark.parametrize('name', soft_suite.fixture_names())
def test_soft_td_fixtures_compiled(name):
    """the M-DQN / SQL / discrete-SAC golden set: bit-identical to eager (within the suite's tolerance where the case
    runs a torch criterion), within tests/test_soft_td.py's tolerance of the stored reference values"""
    case, t, want = soft_suite.load_fixture(name)
    compiled = _CompiledAPI('m_q_1step_td_error', 'q_nstep_sql_td_error', 'q_v_1step_td_error')
    eager = soft_suite.run(api, case, t, 'cuda')
    got = soft_suite.run(compiled, case, t, 'cuda')
    if _torch_callables(case):
        soft_suite.compare(got, eager)
    else:
        _same_bits(got, eager)
    soft_suite.compare(got, want)


@pytest.mark.gpu
@pytest.mark.parametrize('name', sorted(fraction_suite.CASES))
def test_fqf_fraction_fixtures_compiled(name):
    """FQF's fraction loss on its golden set, at both upstream gradients of tests/test_fqf_fraction.py: bit-identical to
    eager, and within that suite's tolerances of the stored reference values"""
    _, t, d = fraction_suite.load_fixture(name)
    compiled = _CompiledAPI('fqf_calculate_fraction_loss')
    for u in fraction_suite.UPSTREAM:
        eager = fraction_suite.run(api, t, 'cuda', u)
        got = fraction_suite.run(compiled, t, 'cuda', u)
        _same_bits(got, eager)
        fraction_suite.close_loss(got['loss'], d['out_loss'])
        if u == 1.0:
            fraction_suite.same_bits(got['grad'], d['out_grad_u1'])
        else:
            assert np.allclose(got['grad'], d['out_grad_u037'], rtol=3e-7, atol=0, equal_nan=True)


@pytest.mark.gpu
@pytest.mark.parametrize('name', ('dqfd_nstep_td_error[is_expert_scalar]', 'dqfd_nstep_td_error_sequence',
                                  'q_nstep_td_error_sequence[ngu]', 'm_q_1step_td_error',
                                  'q_nstep_sql_td_error[value_gamma_scalar]', 'fqf_calculate_fraction_loss'))
def test_reduce_overhead_replays_bit_identical_to_eager(name, monkeypatch):
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
        args = _on_cuda(inputs(_g(100 + step)))
        got = _results(compiled(*args), args)
        args = _on_cuda(inputs(_g(100 + step)))
        want = _results(fn(*args), args)
        assert len(got) == len(want)
        for a, b in zip(got, want):
            assert torch.equal(a, b), (name, step)
        if step == 1:
            allocated.clear()
    assert allocated == [], 'a workspace, record or constant was allocated after warm-up'


@pytest.mark.gpu
@pytest.mark.parametrize('name', ('dqfd_nstep_td_error', 'm_q_1step_td_error'))
def test_dynamic_batch_does_not_recompile(name):
    from torch._dynamo.utils import counters
    torch._dynamo.reset()
    counters.clear()
    fn = torch.compile(CASES[name][1], fullgraph=True)

    def args(S, seed):
        g = _g(seed)
        q, nq, nq1 = (torch.randn(S, 6, generator=g).cuda() for _ in range(3))
        act, nact, nact1 = (torch.randint(0, 6, (S, ), generator=g).cuda() for _ in range(3))
        reward = torch.randn(S, generator=g).cuda() if name == 'm_q_1step_td_error' else \
            torch.randn(NSTEP, S, generator=g).cuda()
        done = (torch.rand(S, generator=g) < 0.2).float().cuda()
        weight, expert = torch.rand(S, generator=g).cuda(), (torch.rand(S, generator=g) < 0.5).float().cuda()
        ts = (q, nq, nq1, act, nact, nact1, reward, done, weight, expert)
        for t in ts:
            torch._dynamo.mark_dynamic(t, t.dim() - 1 if t is reward else 0)
        q.requires_grad_(True)
        if name == 'm_q_1step_td_error':
            return (api.m_q_1step_td_data(q, nq1, nq, act, reward, done, weight), )
        return (api.dqfd_nstep_td_data(q, nq, act, nact, reward, done, done, weight, nq1, nact1, expert), )

    for S in (64, 320):
        a = args(S, S)
        want = _results(CASES[name][1](*a), a)
        got = _results(fn(*a), a)
        for x, y in zip(got, want):
            assert torch.equal(x, y), S
    assert counters['stats']['unique_graphs'] == 1, dict(counters['stats'])


# ---------------------------------------------------------------------------------------------------------------------
# learner steps, model included
# ---------------------------------------------------------------------------------------------------------------------
def _mlp(i, o):
    return nn.Sequential(nn.Linear(i, 64), nn.ReLU(), nn.Linear(64, o)).cuda()


def _dqfd_step():
    """DQfDPolicy's learner step (ding/policy/dqfd.py): the n-step, 1-step and margin losses on an MLP; the per-sample
    error (priorities) and the statistics leave detached"""
    torch.manual_seed(3)
    A, n = 6, 64
    net, target = _mlp(16, A), _mlp(16, A)
    obs, nobs, nobs1 = (torch.randn(n, 16, device='cuda') for _ in range(3))
    act = torch.randint(0, A, (n, ), device='cuda')
    reward, done = torch.randn(3, n, device='cuda'), (torch.rand(n, device='cuda') < 0.1).float()
    expert, weight = (torch.rand(n, device='cuda') < 0.5).float(), torch.rand(n, device='cuda')

    def step(obs, nobs, nobs1, act, reward, done, expert, weight):
        q = net(obs)
        with torch.no_grad():
            nq, nq1 = target(nobs), target(nobs1)
            nact, nact1 = net(nobs).argmax(-1), net(nobs1).argmax(-1)
        loss, td, stats = api.dqfd_nstep_td_error(
            api.dqfd_nstep_td_data(q, nq, act, nact, reward, done, done, weight, nq1, nact1, expert), 0.99, 1.0, 1.0, 0.8,
            nstep=3)
        return loss, td.detach(), torch.stack(stats).detach()
    return step, (obs, nobs, nobs1, act, reward, done, expert, weight), list(net.parameters())


def _r2d2_step():
    """R2D2's per-step loop over a (T, B, N) q sequence in one call, value rescaling on"""
    torch.manual_seed(4)
    A, Ts, n = 6, 10, 16
    net = _mlp(12, A)
    obs, nobs = torch.randn(Ts, n, 12, device='cuda'), torch.randn(Ts, n, 12, device='cuda')
    act = torch.randint(0, A, (Ts, n), device='cuda')
    reward, done = torch.randn(Ts, 5, n, device='cuda'), (torch.rand(Ts, n, device='cuda') < 0.05).float()
    weight = torch.rand(Ts, n, device='cuda')

    def step(obs, nobs, act, reward, done, weight):
        q = net(obs)
        with torch.no_grad():
            nq = net(nobs)
            nact = nq.argmax(-1)
        loss, prio, td = api.q_nstep_td_error_sequence(
            api.q_nstep_td_seq_data(q, nq, act, nact, reward, done, weight), 0.997, nstep=5, rescale=True)
        return loss, prio, td.detach()
    return step, (obs, nobs, act, reward, done, weight), list(net.parameters())


def _fqf_step():
    """FQFPolicy's learner step (ding/policy/fqf.py): the fraction proposal makes the quantiles, the quantile TD loss
    trains the value net at their midpoints and the fraction loss trains the proposal, in one graph"""
    torch.manual_seed(5)
    A, n, Nq, E = 6, 32, 32, 16
    body, frac, embed, head = nn.Linear(8, 64).cuda(), nn.Linear(64, Nq).cuda(), nn.Linear(E, 64).cuda(), \
        nn.Linear(64, A).cuda()
    obs, nobs = torch.randn(n, 8, device='cuda'), torch.randn(n, 8, device='cuda')
    act = torch.randint(0, A, (n, ), device='cuda')
    reward, done = torch.randn(3, n, device='cuda'), (torch.rand(n, device='cuda') < 0.1).float()
    freqs = torch.arange(1, E + 1, device='cuda', dtype=torch.float32) * math.pi

    def quantile_values(feat, tau):  # (B, h), (B, k) -> (B, k, A)
        return head(torch.relu(feat[:, None, :] * embed(torch.cos(tau[..., None] * freqs))))

    def step(obs, nobs, act, reward, done):
        feat = torch.relu(body(obs))
        p = torch.softmax(frac(feat.detach()), -1)
        quantiles = torch.cat([torch.zeros_like(p[:, :1]), p.cumsum(-1)], -1)  # (B, N+1)
        hats = ((quantiles[:, 1:] + quantiles[:, :-1]) / 2).detach()
        q = quantile_values(feat, hats)
        with torch.no_grad():
            nq = quantile_values(torch.relu(body(nobs)), hats)
            nact = nq.mean(1).argmax(-1)
            q_tau_i = quantile_values(feat, quantiles[:, 1:-1])
        td_loss, td = api.fqf_nstep_td_error(api.fqf_nstep_td_data(q, nq, act, nact, reward, done, hats, None), 0.99,
                                             nstep=3)
        fraction_loss = api.fqf_calculate_fraction_loss(q_tau_i, q, quantiles, act)
        return td_loss + fraction_loss, td.detach()
    params = [p for m in (body, frac, embed, head) for p in m.parameters()]
    return step, (obs, nobs, act, reward, done), params


def _sac_discrete_step():
    """SACDiscretePolicy's twin critic (ding/policy/sac.py): one q_v_1step_td_error per Q head against the soft target"""
    torch.manual_seed(6)
    A, n = 6, 128
    q1, q2 = _mlp(10, A), _mlp(10, A)
    obs = torch.randn(n, 10, device='cuda')
    act = torch.randint(0, A, (n, ), device='cuda')
    target_v, reward = torch.randn(n, device='cuda'), torch.randn(n, device='cuda')
    done = (torch.rand(n, device='cuda') < 0.1).float()

    def step(obs, act, target_v, reward, done):
        losses = [api.q_v_1step_td_error(api.q_v_1step_td_data(q(obs), target_v, act, reward, done, None), 0.99)[0]
                  for q in (q1, q2)]
        return losses[0] + losses[1]
    return step, (obs, act, target_v, reward, done), list(q1.parameters()) + list(q2.parameters())


def _mdqn_step():
    """MDQNPolicy's learner step (ding/policy/mdqn.py): the Munchausen target from the target net on both observations"""
    torch.manual_seed(7)
    A, n = 6, 64
    net, target = _mlp(16, A), _mlp(16, A)
    obs, nobs = torch.randn(n, 16, device='cuda'), torch.randn(n, 16, device='cuda')
    act = torch.randint(0, A, (n, ), device='cuda')
    reward, done = torch.randn(n, device='cuda'), (torch.rand(n, device='cuda') < 0.1).float()

    def step(obs, nobs, act, reward, done):
        q = net(obs)
        with torch.no_grad():
            tq, nq = target(obs), target(nobs)
        loss, td, gap, clip = api.m_q_1step_td_error(api.m_q_1step_td_data(q, tq, nq, act, reward, done, None), 0.99,
                                                     0.03, 0.9)
        return loss, td.detach(), gap, clip
    return step, (obs, nobs, act, reward, done), list(net.parameters())


@pytest.mark.gpu
@pytest.mark.parametrize('make', (_dqfd_step, _r2d2_step, _fqf_step, _sac_discrete_step, _mdqn_step),
                         ids=('dqfd', 'r2d2', 'fqf', 'sac_discrete_twin_critic', 'mdqn'))
def test_learner_step_compiles_without_a_graph_break(make):
    """the step's forward (model + loss) compiles as one graph; its backward runs the compiled backward graph"""
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
