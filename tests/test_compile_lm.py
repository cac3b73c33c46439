"""torch.compile over the language-model losses: grpo_policy_error, rloo_policy_error (a built-in or a custom
log_prob_fn), the three log-prob methods, and ppo_policy_error / ppo_error / a2c_error on (B, S, V) token rows.

Under compile these run on the ``b200rl`` custom ops of ``torch_ops``, which recompute the gradient in the backward op
from the per-row values the forward op saved: the forward launch writes no gradient, and the backward launch writes a
fresh buffer (no (B, S, V) copy anywhere).

CPU part: against the logging stand-in for the CUDA library of ``tests/test_launch_log.py``, each loss compiles with
``fullgraph=True``; its forward makes the eager call's C-ABI call with the same int and float arguments, minus the
gradient buffers and the upstream-gradient record; its backward launch is the eager backward's recompute form, reading
the forward's per-row values into a buffer no earlier launch wrote.

GPU part: ``torch.library.opcheck`` on every new op; inductor bit-identical to eager on the golden cases and within the
suites' tolerances of the reference's fixtures; a changing loss mix, a repeated backward and accumulation into .grad;
dynamic B and S without recompiling; ``mode="reduce-overhead"`` replays; a bf16 lm_head in the same graph; peak memory.
"""
import contextlib
import os

import numpy as np
import pytest
import torch
import torch._dynamo

import di_engine_b200 as b2
from di_engine_b200 import ops
from tests import grpo_oracle as go
from tests import ppo_lm_oracle as po
from tests.golden import make_a2c_lm_golden as mk
from tests.test_compile import _launches, _recording, _stand_in

api = b2.rl_utils
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
NEW_OPS = ('token_logp', 'vocab_bwd', 'lm_policy_fwd', 'token_head_fwd', 'ppo_lm_fwd', 'ppo_lm_bwd', 'a2c_lm_fwd',
           'a2c_lm_bwd', 'ppo_value_fwd')


@pytest.fixture(autouse=True)
def _distribution_validation():
    """dynamo turns off torch.distributions' argument validation for the whole process the first time it runs; the
    reference's errors that other tests check depend on it"""
    validate = torch.distributions.Distribution._validate_args
    yield
    torch.distributions.Distribution.set_default_validate_args(validate)


def _g(seed):
    return torch.Generator().manual_seed(seed)


def custom_logp(logits, index):
    """a log_prob_fn of the caller's own: torch ops, traced into the same graph"""
    return torch.log_softmax(logits.float(), -1).gather(-1, index.unsqueeze(-1)).squeeze(-1)


# ---------------------------------------------------------------------------------------------------------------------
# the losses: inputs (B, S, V) in a dtype, and the scalar each backward starts from
# ---------------------------------------------------------------------------------------------------------------------
def _logits(g, B, S, V, dtype, n):
    x = torch.randn(B, S, V, generator=g)
    return [x.to(dtype).requires_grad_(True)] + [(x + 0.1 * torch.randn(B, S, V, generator=g)).to(dtype)
                                                 for _ in range(n - 1)]


def _grpo(dtype, B=2, S=3, V=1024, fn=None, seed=0, dev='cpu'):
    g = _g(seed)
    ln, lo, lr = _logits(g, B, S, V, dtype, 3)
    w = (torch.rand(B, S, generator=g) > 0.3).float()
    w[:, 0] = 1.0  # no sequence whose weights sum to 0 (a NaN loss, which opcheck cannot compare)
    data = api.grpo_policy_data(ln, lo, lr, torch.randint(0, V, (B, S), generator=g), torch.randn(B, generator=g), w)
    data = _to(data, dev)
    return data, (lambda f: f(data, fn or api.efficient_method)), (lambda r: r[0]), [data.logit_new]


def _rloo(dtype, B=4, S=3, V=1024, fn=None, seed=0, dev='cpu'):
    g = _g(seed)
    ln, lo = _logits(g, B, S, V, dtype, 2)
    data = api.rloo_policy_data(ln, lo, torch.randint(0, V, (B, S), generator=g), torch.randn(2, B // 2, generator=g),
                                torch.rand(B, S, generator=g))
    data = _to(data, dev)
    return data, (lambda f: f(data, fn or api.naive_method)), (lambda r: r[0]), [data.logit_new]


def _logp(dtype, B=2, S=3, V=1024, fn=None, seed=0, dev='cpu'):
    g = _g(seed)
    x = _logits(g, B, S, V, dtype, 1)[0]
    idx = torch.randint(0, V, (B, S), generator=g)
    w = torch.randn(B, S, generator=g)
    x, idx, w = _to(x, dev), _to(idx, dev), _to(w, dev)
    return (x, idx), (lambda f: f(x, idx)), (lambda r: (r * w).sum()), [x]


def _ppo_policy(dtype, B=2, S=3, V=1024, fn=None, seed=0, dev='cpu', mix=(1.0, -0.01, 0.1)):
    g = _g(seed)
    ln, lo, lp = _logits(g, B, S, V, dtype, 3)
    data = api.ppo_policy_data(ln, lo, torch.randint(0, V, (B, S), generator=g), torch.randn(B, S, generator=g),
                               torch.rand(B, S, generator=g), lp)
    data = _to(data, dev)
    return data, (lambda f: f(data, kl_type='k3')), (
        lambda r: mix[0] * r[0].policy_loss + mix[1] * r[0].entropy_loss + mix[2] * r[0].kl_div), [data.logit_new]


def _ppo(dtype, B=2, S=3, V=1024, fn=None, seed=0, dev='cpu', mix=(1.0, 0.5, -0.01, 0.1)):
    g = _g(seed)
    ln, lo, lp = _logits(g, B, S, V, dtype, 3)
    vn = torch.randn(B, S, generator=g).requires_grad_(True)
    data = api.ppo_data(ln, lo, torch.randint(0, V, (B, S), generator=g), vn,
                        *(torch.randn(B, S, generator=g) for _ in range(3)), torch.rand(B, S, generator=g), lp)
    data = _to(data, dev)

    def loss(r):
        ls = r[0]
        return mix[0] * ls.policy_loss + mix[1] * ls.value_loss + mix[2] * ls.entropy_loss + mix[3] * ls.kl_div

    return data, (lambda f: f(data)), loss, [data.logit_new, data.value_new]


def _a2c(dtype, B=2, S=3, V=1024, fn=None, seed=0, dev='cpu', mix=(1.0, 0.5, -0.01)):
    g = _g(seed)
    x = _logits(g, B, S, V, dtype, 1)[0]
    v = torch.randn(B, S, generator=g).to(dtype).requires_grad_(True)
    data = api.a2c_data(x, torch.randint(0, V, (B, S), generator=g), v,
                        *(torch.randn(B, S, generator=g) for _ in range(2)), torch.rand(B, S, generator=g))
    data = _to(data, dev)
    return data, (lambda f: f(data)), (
        lambda r: mix[0] * r.policy_loss + mix[1] * r.value_loss + mix[2] * r.entropy_loss), [data.logit, data.value]


def _to(x, dev):
    if isinstance(x, torch.Tensor):
        return x.detach().to(dev).requires_grad_(x.requires_grad)
    if isinstance(x, tuple) and hasattr(x, '_fields'):
        return type(x)(*[_to(y, dev) for y in x])
    return x


# name -> (case builder, public function, takes a log_prob_fn)
LOSSES = {
    'grpo_policy_error': (_grpo, 'grpo_policy_error', True),
    'rloo_policy_error': (_rloo, 'rloo_policy_error', True),
    'efficient_method': (_logp, 'efficient_method', False),
    'ppo_policy_error': (_ppo_policy, 'ppo_policy_error', False),
    'ppo_error': (_ppo, 'ppo_error', False),
    'a2c_error': (_a2c, 'a2c_error', False),
}
DTYPES = {'f32': torch.float32, 'bf16': torch.bfloat16}
CPU_CASES = [(n, d, c) for n in LOSSES for d in DTYPES for c in ((False, True) if LOSSES[n][2] else (False, ))]


def _case_id(c):
    return '%s-%s%s' % (c[0], c[1], '-custom' if c[2] else '')


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the launch sequence of the compiled loss against the stand-in library
# ---------------------------------------------------------------------------------------------------------------------
# the recompute form of a launch: argument index -> its value under compile, for the vocabulary entry points whose eager
# forward writes gradients (the buffers, the record it reads and the one it writes) and whose eager backward verifies
# them (the forward's record and the call site's record; GRPO / RLOO: the unit-upstream skip)
_RECOMPUTE = {
    'b200rl_grpo_fwd_grad': {15: True},
    'b200rl_rloo_fwd_grad': {14: True},
    'b200rl_ppo_lm_fwd_grad': {13: True, 14: True, 20: True},
    'b200rl_a2c_lm_fwd_grad': {9: True, 10: True, 16: True, 17: True},
    'b200rl_ppo_lm_bwd': {13: True, 14: True},
    'b200rl_a2c_lm_bwd': {13: True, 14: True},
    'b200rl_token_logp_bwd': {6: 0},
}
# the argument indices of each backward launch: (its gradient buffers, the forward's per-row values it reads; the
# log-prob methods' coefficient is their upstream gradient)
_BWD_ARGS = {
    'b200rl_token_logp_bwd': ((9, ), (3, )),
    'b200rl_ppo_lm_bwd': ((15, ), (6, 7, 8, 9)),
    'b200rl_a2c_lm_bwd': ((15, 16), (6, 7, 8, 9)),
}


def _recompute(launches):
    out = []
    for fn, check, args in launches:
        args = list(args)
        for i, v in _RECOMPUTE.get(fn, {}).items():
            args[i] = v
        out.append((fn, check, args))
    return out


def _step(name, dtype, custom, f=None):
    build, public, _ = LOSSES[name]
    data, call, loss, _ = build(DTYPES[dtype], fn=custom_logp if custom else None)
    with _stand_in() as log:
        loss(call(f or getattr(api, public))).backward()
    return log


@pytest.mark.filterwarnings('ignore:invalid value encountered in cast')  # the stand-in leaves outputs uninitialised
@pytest.mark.parametrize('case', CPU_CASES, ids=_case_id)
def test_compiled_launch_sequence_is_the_recompute_form_of_eager(case):
    name, dtype, custom = case
    torch._dynamo.reset()
    want = _step(name, dtype, custom)
    got = _step(name, dtype, custom, torch.compile(getattr(api, LOSSES[name][1]), backend='aot_eager', fullgraph=True))
    assert len(want) > 0
    assert _launches(got) == _recompute(_launches(want))
    # the backward launch reads the forward's per-row values and writes buffers no forward launch was given
    fwd_labels = {a for e in got if e['fn'] not in _BWD_ARGS and e['fn'] != 'b200rl_scale' for a in e['args']}
    for e in got:
        if e['fn'] in _BWD_ARGS:
            outs, saved = _BWD_ARGS[e['fn']]
            assert all(e['args'][i] not in fwd_labels for i in outs), e
            assert all(e['args'][i] in fwd_labels for i in saved if e['args'][i] is not None), e


def test_new_ops_schemas_hold_only_tensors_and_scalars():
    for name in NEW_OPS:
        schema = getattr(torch.ops.b200rl, name).default._schema
        for a in schema.arguments:
            assert str(a.type) in ('Tensor', 'Optional[Tensor]', 'SymInt', 'int', 'float', 'bool', 'str'), (
                name, a.name, a.type)
        assert not any(a.alias_info is not None for a in schema.arguments), name


def test_fake_kernels_keep_the_logits_dtype_and_symbolic_rows():
    from torch._subclasses.fake_tensor import FakeTensorMode
    from torch.fx.experimental.symbolic_shapes import ShapeEnv
    with FakeTensorMode(shape_env=ShapeEnv()) as mode:
        x = mode.from_tensor(torch.empty(2, 3, 8, dtype=torch.bfloat16), symbolic_context=None)
        rows = torch.empty(6)
        grad = torch.ops.b200rl.vocab_bwd(x.view(6, 8), rows.long(), rows, rows, None)
        assert grad.dtype == torch.bfloat16
        out = torch.ops.b200rl.ppo_lm_fwd(x, x, None, rows.long(), rows, None, 0.2, 0.0, 1, True)
        assert [t.dtype for t in out] == [torch.float32] * 5 and out[1].shape == (6, ) and out[4].shape == (0, )


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
DEV = 'cuda:0'


@contextlib.contextmanager
def _lazy_info():
    """the monitors stay on the device: a python float leaves an inductor graph through a CPU kernel, which needs a host
    C++ toolchain with OpenMP"""
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(api.ppo, 'LAZY_INFO', True)
        yield


@contextlib.contextmanager
def _eager_recomputes():
    """Eager ppo_policy_error / a2c_error take the forward-written gradient when the upstream gradients match their
    record, and recompute otherwise; the two branches may round the kl term differently in the last bit.  Under compile
    the gradient is always recomputed, so the eager side of a bit-for-bit comparison is made to recompute too, by a
    record no upstream gradient matches."""
    saved = {k: h.clone() for k, h in ops._HINT.items()}
    for kind in ('policy', 'ppo', 'a2c'):
        ops.ppo_hint(torch.device(DEV), kind).fill_(float('nan'))
    yield
    for k, h in ops._HINT.items():
        h.copy_(saved[k] if k in saved else torch.tensor(ops._HINT_INIT[k[1]]))


def _results(out, grads):
    flat = [x for x in torch.utils._pytree.tree_leaves(out) if x is not None]
    return [torch.as_tensor(x).detach().clone().cpu() for x in flat] + [g.detach().clone().cpu() for g in grads]


def _run(f, call, loss, leaves, twice=False, mix2=None):
    out = call(f)
    total = loss(out)
    grads = torch.autograd.grad(total, leaves, retain_graph=twice)
    res = _results(out, grads)
    if twice:
        res += [g.cpu() for g in torch.autograd.grad(mix2(out) if mix2 else total, leaves)]
    return res


def _assert_same(got, want, what):
    assert len(got) == len(want), what
    for i, (a, b) in enumerate(zip(got, want)):
        assert a.dtype == b.dtype and a.shape == b.shape, (what, i)
        assert torch.equal(a, b) or (a.is_floating_point() and torch.equal(a.isnan(), b.isnan()) and
                                     torch.equal(a[~a.isnan()], b[~b.isnan()])), (what, i)


def _golden_cases():
    out = []
    for name, c in go.CASES.items():
        if c[3] < 2 ** 17:  # the V = 152k cases take the same code path as V = 32771 and cost seconds to compile around
            out.append(('lm_policy', name))
    out += [('ppo_lm', n) for n in po.CASES] + [('a2c_lm', n) for n in mk.CASES]
    return out


def _golden_call(kind, name):
    """(inputs on the GPU, the call, the loss, the leaves, the fixture's values and tolerance)"""
    if kind == 'lm_policy':
        d = {k: (v.to(DEV) if isinstance(v, torch.Tensor) else v) for k, v in go.make_case(name).items()}
        d['logit_new'].requires_grad_(True)
        grpo = go.CASES[name][0] == 'grpo'

        def call(f):
            if grpo:
                return f['grpo'](api.grpo_policy_data(d['logit_new'], d['logit_old'], d['logit_ref'], d['action'],
                                                      d['adv'], d['weight']), api.efficient_method, go.CLIP, go.BETA)
            return f['rloo'](api.rloo_policy_data(d['logit_new'], d['logit_old'], d['action'], d['reward'], d['weight']),
                             api.efficient_method, go.CLIP)

        gold = np.load(os.path.join(GOLD, 'grpo_rloo', name + '.npz'))
        bf16 = go.CASES[name][5] == torch.bfloat16
        # clipfrac on bf16 logits: test_grpo_rloo.py's bar (the reference rounds the ratio to bf16 before the clip test)
        return call, (lambda r: r[0]), [d['logit_new']], (lambda r: (r[0], r[1].approx_kl, r[1].clipfrac)), (
            gold['loss'], gold['approx_kl'], gold['clipfrac']), (2e-2, 2e-2, 0.1) if bf16 else 1e-5
    if kind == 'ppo_lm':
        d = po.make_case(name, DEV)
        d['logit_new'].requires_grad_(True)
        kw = dict(zip(('dual_clip', 'kl_type', 'entropy_bonus'), po.case_args(name)))
        has_kl = d['logit_pretrained'] is not None

        def call(f):
            return f['ppo_policy'](api.ppo_policy_data(d['logit_new'], d['logit_old'], d['action'], d['adv'],
                                                       d['weight'], d['logit_pretrained']), clip_ratio=po.CLIP, **kw)

        def loss(r):
            total = po.MIX[0] * r[0].policy_loss
            if kw.get('entropy_bonus', True):
                total = total + po.MIX[1] * r[0].entropy_loss
            return total + po.MIX[2] * r[0].kl_div if has_kl else total

        gold = np.load(os.path.join(GOLD, 'ppo_lm', name + '.npz'))
        bf16 = po.CASES[name][0] == torch.bfloat16
        return call, loss, [d['logit_new']], (lambda r: (r[0].policy_loss, r[0].kl_div, r[1].approx_kl)), (
            gold['policy'], gold['kl'], gold['approx_kl']), 2e-2 if bf16 else 1e-5
    d = mk.make_case(name, DEV)
    d['logit'].requires_grad_(True)
    d['value'].requires_grad_(True)

    def call(f):
        return f['a2c'](api.a2c_data(d['logit'], d['action'], d['value'], d['adv'], d['return_'], d['weight']))

    gold = np.load(os.path.join(GOLD, 'a2c_lm', name + '.npz'))
    bf16 = mk.CASES[name][0] == torch.bfloat16
    return call, (lambda r: mk.MIX[0] * r.policy_loss + mk.MIX[1] * r.value_loss + mk.MIX[2] * r.entropy_loss), [
        d['logit'], d['value']], (lambda r: tuple(r)), (gold['policy'], gold['value'], gold['entropy']), (
            2e-2 if bf16 else 1e-5)


def _ppo_policy_on_device(data, **kw):
    """ppo_policy_error without the reference's CPU ``torch.tensor(0.0)`` entropy of a call without the entropy bonus: a
    CPU tensor leaves an inductor graph through a CPU kernel, which needs a host C++ toolchain with OpenMP"""
    loss, info = api.ppo_policy_error(data, **kw)
    entropy = loss.entropy_loss if kw.get('entropy_bonus', True) else None
    return api.ppo_policy_loss(loss.policy_loss, entropy, loss.kl_div), info


EAGER = {'grpo': api.grpo_policy_error, 'rloo': api.rloo_policy_error, 'ppo_policy': _ppo_policy_on_device,
         'a2c': api.a2c_error}


@pytest.fixture
def compiled():
    torch._dynamo.reset()
    return {k: torch.compile(f, fullgraph=True) for k, f in EAGER.items()}


@pytest.mark.gpu
@pytest.mark.parametrize('case', _golden_cases(), ids=lambda c: '%s-%s' % c)
def test_inductor_bit_identical_to_eager_and_within_fixture_tolerance(case, compiled):
    call, loss, leaves, values, fixture, tol = _golden_call(*case)
    with _lazy_info(), pytest.MonkeyPatch.context() as mp:
        # as the suites do: fp32 calls below LM_MIN_VOCAB take the vocabulary kernel too, so that V = 1000 / 1003 test it
        mp.setattr(api.ppo, 'LM_MIN_VOCAB', 1)
        got = _run(compiled, call, loss, leaves)
        with _eager_recomputes():
            want = _run(EAGER, call, loss, leaves)
        out = call(compiled)
        vals = [float(x.detach()) if isinstance(x, torch.Tensor) else float(x) for x in values(out)]
    _assert_same(got, want, case)
    tol = np.broadcast_to(np.asarray(tol, np.float64), (len(vals), ))
    want_vals = np.asarray([float(x) for x in fixture])
    assert np.all((np.abs(np.asarray(vals) - want_vals) <= tol + tol * np.abs(want_vals)) |
                  (np.isnan(vals) & np.isnan(want_vals))), (vals, want_vals, tol)


@pytest.mark.gpu
@pytest.mark.parametrize('name', NEW_OPS)
def test_opcheck(name):
    mode, calls = _recording()
    runs = {
        'token_logp': lambda: _logp(torch.bfloat16, dev=DEV), 'vocab_bwd': lambda: _grpo(torch.float32, dev=DEV),
        'lm_policy_fwd': lambda: _rloo(torch.bfloat16, dev=DEV),
        'token_head_fwd': lambda: _grpo(torch.float32, fn=custom_logp, dev=DEV),
        'ppo_lm_fwd': lambda: _ppo_policy(torch.bfloat16, dev=DEV), 'ppo_lm_bwd': lambda: _ppo_policy(torch.float32,
                                                                                                       dev=DEV),
        'a2c_lm_fwd': lambda: _a2c(torch.bfloat16, dev=DEV), 'a2c_lm_bwd': lambda: _a2c(torch.float32, dev=DEV),
        'ppo_value_fwd': lambda: _ppo(torch.float32, dev=DEV)}
    data, call, loss, leaves = runs[name]()
    with mode, pytest.MonkeyPatch.context() as mp:
        mp.setattr(torch.compiler, 'is_compiling', lambda: True)  # the traced path, run eagerly
        mp.setattr(api.ppo, 'LAZY_INFO', True)
        loss(call(getattr(api, {'token_logp': 'efficient_method', 'vocab_bwd': 'grpo_policy_error',
                                'lm_policy_fwd': 'rloo_policy_error', 'token_head_fwd': 'grpo_policy_error',
                                'ppo_lm_fwd': 'ppo_policy_error', 'ppo_lm_bwd': 'ppo_policy_error',
                                'a2c_lm_fwd': 'a2c_error', 'a2c_lm_bwd': 'a2c_error',
                                'ppo_value_fwd': 'ppo_error'}[name]))).backward()
    found = [(op, a, k) for op, a, k in calls if op._opname == name]
    assert found, [op._opname for op, _, _ in calls]
    op, a, k = found[0]
    if name.endswith('_bwd'):  # a backward op is not differentiated again
        a, k = torch.utils._pytree.tree_map_only(torch.Tensor, lambda x: x.detach(), (a, k))
    torch.library.opcheck(op, a, k)


@pytest.mark.gpu
def test_changing_loss_mix_stays_exact():
    torch._dynamo.reset()
    with _lazy_info():
        for public, build, mixes in (
                ('ppo_error', _ppo, [(1.0, 0.5, -0.01, 0.1), (1.0, 0.5, -0.05, 0.1), (1.0, 0.5, 0.0, 0.1),
                                     (1.0, 0.5, -0.01, 0.1)]),
                ('a2c_error', _a2c, [(1.0, 0.5, -0.01), (1.0, 1.0, -0.01), (1.0, 0.25, -0.01), (1.0, 0.5, -0.01)])):
            f = torch.compile(getattr(api, public), fullgraph=True)
            for i, mix in enumerate(mixes):
                for dtype in (torch.float32, torch.bfloat16):
                    _, call, loss, leaves = build(dtype, B=4, S=16, V=4099, seed=i, dev=DEV, mix=mix)
                    got = _run(f, call, loss, leaves)
                    with _eager_recomputes():
                        want = _run(getattr(api, public), call, loss, leaves)
                    _assert_same(got, want, (public, mix, dtype))


@pytest.mark.gpu
@pytest.mark.parametrize('name', ('grpo_policy_error', 'ppo_policy_error', 'a2c_error'))
def test_repeated_backward_and_accumulation_stay_exact(name):
    """retain_graph: a second backward with the same and with different loss weights; and .grad accumulating over
    calls that start from an existing .grad"""
    build, public, _ = LOSSES[name]
    torch._dynamo.reset()
    f = torch.compile(getattr(api, public), fullgraph=True)
    with _lazy_info():
        for dtype in (torch.float32, torch.bfloat16):
            _, call, loss, leaves = build(dtype, B=4, S=8, V=2053, dev=DEV)

            def scaled(r):
                return 0.5 * loss(r)

            for mix2 in (None, scaled):
                got = _run(f, call, loss, leaves, twice=True, mix2=mix2)
                with _eager_recomputes():
                    want = _run(getattr(api, public), call, loss, leaves, twice=True, mix2=mix2)
                _assert_same(got, want, (name, dtype, mix2))

            def accumulate(fn):
                for x in leaves:
                    x.grad = torch.full_like(x, 0.25)
                for _ in range(2):
                    loss(call(fn)).backward()
                return [x.grad.clone().cpu() for x in leaves]

            got = accumulate(f)
            with _eager_recomputes():
                want = accumulate(getattr(api, public))
            _assert_same(got, want, (name, dtype, 'accumulate'))
            for x in leaves:
                x.grad = None


@pytest.mark.gpu
@pytest.mark.parametrize('name', ('grpo_policy_error', 'rloo_policy_error', 'efficient_method', 'ppo_error',
                                  'a2c_error'))
def test_dynamic_batch_and_length_do_not_recompile(name):
    from torch._dynamo.utils import counters
    build, public, _ = LOSSES[name]
    torch._dynamo.reset()
    counters.clear()
    f = torch.compile(getattr(api, public), fullgraph=True)
    with _lazy_info():
        for B, S in ((4, 5), (6, 11), (8, 17)):
            data, call, loss, leaves = build(torch.bfloat16, B=B, S=S, V=1031, seed=S, dev=DEV)
            for t in torch.utils._pytree.tree_leaves(data):
                if isinstance(t, torch.Tensor) and t.dim() >= 2 and t.shape[:2] == (B, S):
                    torch._dynamo.mark_dynamic(t, 0)
                    torch._dynamo.mark_dynamic(t, 1)
                elif isinstance(t, torch.Tensor) and t.shape == (B, ):  # GRPO's adv
                    torch._dynamo.mark_dynamic(t, 0)
                elif isinstance(t, torch.Tensor) and t.shape == (2, B // 2):  # RLOO's reward (K, B / K)
                    torch._dynamo.mark_dynamic(t, 1)
            got = _run(f, call, loss, leaves)
            with _eager_recomputes():
                want = _run(getattr(api, public), call, loss, leaves)
            _assert_same(got, want, (name, B, S))
    assert counters['stats']['unique_graphs'] == 1, dict(counters['stats'])


@pytest.mark.gpu
@pytest.mark.parametrize('name', ('grpo_policy_error', 'efficient_method', 'ppo_error', 'a2c_error'))
def test_reduce_overhead_replays_bit_identical_to_eager(name):
    build, public, _ = LOSSES[name]
    torch._dynamo.reset()
    f = torch.compile(getattr(api, public), mode='reduce-overhead', fullgraph=True)
    with _lazy_info():
        for step in range(12):  # 2 warm-up / record calls, then replays
            _, call, loss, leaves = build(torch.bfloat16, B=4, S=16, V=4099, seed=step, dev=DEV)
            got = _run(f, call, loss, leaves)
            with _eager_recomputes():
                want = _run(getattr(api, public), call, loss, leaves)
            _assert_same(got, want, (name, step))


@pytest.mark.gpu
def test_bf16_lm_head_and_grpo_in_one_graph():
    B, S, H, V = 4, 16, 256, 4099
    g = _g(3)
    head = torch.nn.Linear(H, V, bias=False).to(DEV, torch.bfloat16)
    hidden = torch.randn(B, S, H, generator=g).to(DEV, torch.bfloat16)
    old, ref = (torch.randn(B, S, V, generator=g).to(DEV, torch.bfloat16) for _ in range(2))
    act, adv = torch.randint(0, V, (B, S), generator=g).to(DEV), torch.randn(B, generator=g).to(DEV)

    def step(x):
        loss, info = api.grpo_policy_error(api.grpo_policy_data(head(x), old, ref, act, adv, None))
        return loss, info.approx_kl

    torch._dynamo.reset()
    with _lazy_info():
        f = torch.compile(step, fullgraph=True)
        loss, _ = f(hidden)
        loss.backward()
        got = head.weight.grad.clone()
        head.weight.grad = None
        want_loss, _ = step(hidden)
        want_loss.backward()
    assert loss.dtype == torch.float32 and got.dtype == torch.bfloat16
    torch.testing.assert_close(loss, want_loss, rtol=1e-3, atol=1e-3)
    torch.testing.assert_close(got.float(), head.weight.grad.float(), rtol=2e-2, atol=1e-3)


@pytest.mark.gpu
@pytest.mark.parametrize('name', ('grpo_policy_error', 'a2c_error'))
def test_peak_memory_no_more_than_eager_plus_64_mb(name):
    """(B, S, V) fp32 of 1 GiB: the compiled forward + backward holds no (B, S, V) buffer eager does not"""
    build, public, _ = LOSSES[name]
    torch._dynamo.reset()
    f = torch.compile(getattr(api, public), fullgraph=True)
    peaks = {}
    with _lazy_info():
        for mode, fn in (('warm', f), ('eager', getattr(api, public)), ('compiled', f)):
            _, call, loss, leaves = build(torch.float32, B=8, S=1024, V=32768, dev=DEV)
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            grads = torch.autograd.grad(loss(call(fn)), leaves)
            torch.cuda.synchronize()
            peaks[mode] = torch.cuda.max_memory_allocated() - base
            del grads
    assert peaks['compiled'] <= peaks['eager'] + (64 << 20), peaks
