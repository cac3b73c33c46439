"""torch.compile over the language-model losses from the lm_head's hidden states: grpo_policy_error_linear,
rloo_policy_error_linear, ppo_policy_error_linear, a2c_error_linear and token_logp_linear.

Under compile each call is one ``b200rl`` custom op whose body is eager's chunk loop (``ops.lm_chunks_``).  The forward op
writes dH / dW / d value for a unit upstream gradient, as eager's forward does, and the backward op scales them out of
place (``b200rl_lm_linear_scale_out``; A2C's fp32 d value through ``b200rl_scale``) where eager scales in place.

CPU part: against the logging stand-in for the CUDA library of ``tests/test_launch_log.py``, each loss compiles with
``backend='aot_eager', fullgraph=True`` and makes eager's C-ABI launches in eager's order -- one row launch per chunk --
with the out-of-place scale in place of the in-place one, one per wanted gradient and none under ``no_grad``; every
argument error of the eager call is raised while compiling; the new schemas hold tensors and scalars only; every public
language-model function of ``rl_utils`` is in a traced list.

GPU part: ``torch.library.opcheck`` on every new op; inductor bit-identical to eager on several chunks in fp32 and bf16,
under an upstream gradient != 1 and a second backward (both also against float64); ``mode="reduce-overhead"`` replays;
dynamic B and S without recompiling; learner steps with a model in front of the loss that compile with no graph break.
"""
import contextlib

import pytest
import torch
import torch._dynamo
import torch.nn.functional as F

import di_engine_b200 as b2
from di_engine_b200 import ops
from tests import test_compile_lm
from tests import test_lm_linear as tl
from tests import test_lm_linear_pg as tp
from tests.test_compile import _launches, _recording, _stand_in

R = b2.rl_utils
TRACED = ('grpo_policy_error_linear', 'rloo_policy_error_linear', 'ppo_policy_error_linear', 'a2c_error_linear',
          'token_logp_linear')
NEW_OPS = ('lm_linear_loss', 'lm_linear_pg', 'lm_linear_scale_out', 'lm_logp', 'lm_logp_bwd')
# public functions no other suite compiles on their own, that route to ops already traced: name -> inputs


def _value_in(g):
    return (R.ppo_value_data(torch.randn(6, generator=g).requires_grad_(True), torch.randn(6, generator=g),
                             torch.randn(6, generator=g), None), )


def _logp_in(g):
    return torch.randn(2, 3, 1031, generator=g).requires_grad_(True), torch.randint(0, 1031, (2, 3), generator=g)


ALSO_TRACED = {
    'ppo_value_error': _value_in, 'happo_value_error': _value_in, 'naive_method': _logp_in,
    'less_efficient_method': _logp_in,
}


@pytest.fixture(autouse=True, scope='module')
def _leave_no_compiled_state():
    """after the module: no compiled code, CUDA-graph tree or cached block of this module's calls is left for the suites
    that run next (some count the kernels of their own calls)"""
    yield
    torch._dynamo.reset()
    if torch.cuda.is_available():
        from torch._inductor import cudagraph_trees
        cudagraph_trees.reset_cudagraph_trees()
        torch.cuda.synchronize()
        torch.cuda.empty_cache()


@pytest.fixture(autouse=True)
def _distribution_validation():
    """dynamo turns off torch.distributions' argument validation for the whole process the first time it runs"""
    validate = torch.distributions.Distribution._validate_args
    yield
    torch.distributions.Distribution.set_default_validate_args(validate)


# ---------------------------------------------------------------------------------------------------------------------
# the calls: (kind, data on a device) -> (the call's result, the scalar its backward starts from)
# ---------------------------------------------------------------------------------------------------------------------
def _call(kind, d):
    if kind in ('grpo', 'rloo'):
        loss, info = tl.loss_call(kind, d, clip_ratio=tl.go.CLIP, **({'beta': tl.go.BETA} if kind == 'grpo' else {}))
        return (loss, info), loss
    if kind == 'ppo':
        out, info = tp.ppo_call(d, clip_ratio=tp.po.CLIP, kl_type='k3', entropy_weight=tp.EW, kl_weight=tp.KW)
        return (out, info), out.loss
    if kind == 'ppo_dc':  # dual clip, no entropy, no pretrained policy
        out, info = tp.ppo_call(dict(d, logp_pretrained=None), clip_ratio=tp.po.CLIP, dual_clip=2.0, entropy_bonus=False)
        return (out, info), out.loss
    if kind == 'a2c':
        out = tp.a2c_call(d, value_weight=tp.VW, entropy_weight=tp.EW)
        return out, out.loss
    lp = R.token_logp_linear(d['hidden'], d['lm_weight'], d['action'])
    return lp, (lp * d['g']).sum()


KINDS = ('grpo', 'rloo', 'ppo', 'ppo_dc', 'a2c', 'logp')


def _cpu_data(kind, grads):
    d = tl.make(kind) if kind in ('grpo', 'rloo') else tp.make()
    d['g'] = torch.randn(tl.B_, tl.S_, generator=torch.Generator().manual_seed(3))
    d['hidden'].requires_grad_(grads[0])
    d['lm_weight'].requires_grad_(grads[1])
    if kind == 'a2c':
        d['value'].requires_grad_(grads[2])
    return d


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------
@contextlib.contextmanager
def _chunked_stand_in():
    """the stand-in library, 132 SMs and 128-row chunks: 300 rows in chunks of 128, 128 and 44"""
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(ops, 'sm_count', lambda dev: 132)
        mp.setattr(ops, 'LM_CHUNK_BYTES', 128 * tl.V_ * 4)
        with _stand_in() as log:
            yield log


def _step(fn, kind, grads, no_grad=False):
    d = _cpu_data(kind, grads)
    with _chunked_stand_in() as log:
        with torch.no_grad() if no_grad else contextlib.nullcontext():
            _, total = fn(kind, d)
        if total.requires_grad:
            total.backward()
    return log


def _eager_form(launches):
    """eager's launches as the compiled call makes them: each in-place scale of a saved gradient becomes the out-of-place
    scale into a fresh buffer -- b200rl_lm_linear_scale_out for dH / dW, b200rl_scale for A2C's fp32 d value (the last
    scale of a call that wants it) -- with the same dtype, upstream-gradient pointer and element count"""
    out = []
    for fn, check, args in launches:
        if fn == 'b200rl_lm_linear_scale':
            dt, pg, x, n, st = args
            out.append(('b200rl_lm_linear_scale_out', 'b200rl_lm_linear_scale_out', [dt, pg, x, False, n, st]))
        else:
            out.append((fn, check, args))
    return out


def _dv_scale(launches):
    """A2C's d value: eager's last in-place scale (fp32, N elements) is the compiled call's b200rl_scale"""
    fn, check, args = launches[-1]
    assert fn == 'b200rl_lm_linear_scale_out' and args[0] == 0 and args[4] == tl.B_ * tl.S_
    return launches[:-1] + [('b200rl_scale', 'b200rl_scale', [args[1], args[2], False, args[4], args[5]])]


GRADS = [(True, True, False), (True, False, False), (False, True, False), (False, False, True), (True, True, True)]
CPU_CASES = [(k, g) for k in KINDS for g in GRADS if k == 'a2c' or not g[2]]


@pytest.mark.filterwarnings('ignore:invalid value encountered in cast')  # the stand-in leaves outputs uninitialised
@pytest.mark.parametrize('kind,grads', CPU_CASES, ids=lambda c: str(c))
def test_compiled_launches_are_eagers_with_the_out_of_place_scale(kind, grads):
    torch._dynamo.reset()
    want = _launches(_step(lambda k, d: _call(k, d), kind, grads))
    got = _launches(_step(torch.compile(_call, backend='aot_eager', fullgraph=True), kind, grads))
    want = _eager_form(want)
    if kind == 'a2c' and grads[2]:
        want = _dv_scale(want)
    assert got == want
    row = {'logp': 'b200rl_lm_linear_fwd', 'grpo': 'b200rl_lm_linear_fwd',
           'rloo': 'b200rl_lm_linear_fwd'}.get(kind, 'b200rl_lm_linear_pg_fwd')
    assert [a[3:5] for fn, _, a in got if fn == row] == [[0, 128], [128, 128], [256, 44]]  # one row launch per chunk
    n_scales = sum(1 for fn, _, _ in got if fn in ('b200rl_lm_linear_scale_out', 'b200rl_scale'))
    if kind == 'logp':  # its backward recomputes each chunk: no saved gradient to scale
        assert n_scales == 0 and [fn for fn, _, _ in got].count('b200rl_lm_linear_bwd') == 3 * any(grads[:2])
    else:
        assert n_scales == sum(grads[:2]) + (grads[2] and kind == 'a2c')  # one per wanted gradient


@pytest.mark.filterwarnings('ignore:invalid value encountered in cast')
@pytest.mark.parametrize('kind', KINDS)
def test_no_grad_compiled_makes_no_scale_and_no_gradient_buffer(kind):
    torch._dynamo.reset()
    want = _launches(_step(lambda k, d: _call(k, d), kind, (True, True, True), no_grad=True))
    with tl._Ops() as rec:
        got = _launches(_step(torch.compile(_call, backend='aot_eager', fullgraph=True), kind, (True, True, True),
                              no_grad=True))
    assert got == want
    assert not any(fn.endswith(('_scale', '_scale_out')) or fn == 'b200rl_scale' for fn, _, _ in got)
    assert not any(a[22 if kind in ('grpo', 'rloo') else 24] for fn, _, a in got if fn.endswith('_fwd') and kind != 'logp')
    assert (tl.B_ * tl.S_, tl.D_) not in rec.allocated() and (tl.V_, tl.D_) not in rec.allocated()


# each case: (kind, a change to the data or None, the call's keyword options, the error of the eager call)
ERRORS = {
    'rank': ('grpo', lambda d: dict(d, hidden=d['hidden'][0]), {}, RuntimeError),
    'width': ('grpo', lambda d: dict(d, lm_weight=d['lm_weight'][:, :3]), {}, RuntimeError),
    'float64': ('grpo', lambda d: dict(d, hidden=d['hidden'].double(), lm_weight=d['lm_weight'].double()), {}, TypeError),
    'mixed_dtypes': ('rloo', lambda d: dict(d, lm_weight=d['lm_weight'].bfloat16()), {}, TypeError),
    'action_shape': ('grpo', lambda d: dict(d, action=d['action'][:, :5]), {}, RuntimeError),
    'logp_old_shape': ('grpo', lambda d: dict(d, logp_old=d['logp_old'][:, :5]), {}, RuntimeError),
    'adv_count': ('grpo', lambda d: dict(d, adv=d['adv'][:2]), {}, RuntimeError),
    'weight_shape': ('rloo', lambda d: dict(d, weight=d['weight'][:, :5]), {}, RuntimeError),
    'ppo_adv_shape': ('ppo', lambda d: dict(d, adv=d['adv'][:, :5]), {}, RuntimeError),
    'ppo_float16': ('ppo', lambda d: dict(d, hidden=d['hidden'].half(), lm_weight=d['lm_weight'].half()), {}, TypeError),
    'ppo_entropy_weight': ('ppo', None, {'entropy_bonus': False, 'entropy_weight': 0.1}, ValueError),
    'ppo_kl_weight': ('ppo', lambda d: dict(d, logp_pretrained=None), {'kl_weight': 0.1}, ValueError),
    'ppo_kl_type': ('ppo', None, {'kl_type': 'k9'}, ValueError),
    'ppo_dual_clip': ('ppo', None, {'dual_clip': 0.5}, AssertionError),
    'a2c_value_shape': ('a2c', lambda d: dict(d, value=d['value'][:, :5]), {}, RuntimeError),
    'a2c_return_shape': ('a2c', lambda d: dict(d, return_=d['return_'][:2]), {}, RuntimeError),
    'logp_index_shape': ('logp', lambda d: dict(d, action=d['action'][:2]), {}, RuntimeError),
}


def _bad_call(name):
    kind, change, kw, _ = ERRORS[name]
    d = _cpu_data(kind, (True, True, False))
    d = change(d) if change else d
    if kind in ('grpo', 'rloo'):
        return lambda: tl.loss_call(kind, d)
    if kind == 'ppo':
        return lambda: tp.ppo_call(d, **kw)
    if kind == 'a2c':
        return lambda: tp.a2c_call(d)
    return lambda: R.token_logp_linear(d['hidden'], d['lm_weight'], d['action'])


@pytest.mark.filterwarnings('ignore:invalid value encountered in cast')
@pytest.mark.parametrize('name', sorted(ERRORS))
def test_eager_errors_are_raised_while_compiling(name):
    exc = ERRORS[name][3]
    torch._dynamo.reset()
    with _chunked_stand_in():
        with pytest.raises(exc) as eager:
            _bad_call(name)()
        # dynamo stops tracing at the raise and runs the frame as Python, which raises what eager mode raises
        with pytest.raises(exc) as compiled:
            torch.compile(_bad_call(name), backend='aot_eager')()
    assert str(compiled.value).split('\n\nfrom user code:')[0] == str(eager.value)


@pytest.mark.filterwarnings('ignore:invalid value encountered in cast')
@pytest.mark.parametrize('name', sorted(ALSO_TRACED))
def test_functions_on_traced_ops_compile_with_eagers_launches(name):
    fn = getattr(R, name)

    def run(f):
        args = ALSO_TRACED[name](torch.Generator().manual_seed(4))
        with _chunked_stand_in() as log:
            f(*args).sum().backward()
        return _launches(log)

    torch._dynamo.reset()
    want = run(fn)
    assert want and run(torch.compile(fn, backend='aot_eager', fullgraph=True)) == want


def test_new_ops_schemas_hold_only_tensors_and_scalars():
    for name in NEW_OPS:
        schema = getattr(torch.ops.b200rl, name).default._schema
        for a in schema.arguments:
            assert str(a.type) in ('Tensor', 'Optional[Tensor]', 'SymInt', 'int', 'float', 'bool', 'str'), (
                name, a.name, a.type)
        assert not any(a.alias_info is not None for a in schema.arguments), name


def test_fake_kernels_give_wanted_gradients_only():
    from torch._subclasses.fake_tensor import FakeTensorMode
    with FakeTensorMode():
        h, w = torch.empty(300, 8, dtype=torch.bfloat16), torch.empty(1031, 8, dtype=torch.bfloat16)
        rows = torch.empty(300)
        out, dh, dw = torch.ops.b200rl.lm_linear_loss(h, w, rows.long(), rows, rows, torch.empty(3), None, 'grpo', 3, 100,
                                                      1, 0.2, 0.1, True, False)
        assert out.shape == (3, ) and dh.shape == h.shape and dh.dtype == torch.bfloat16 and dw.numel() == 0
        loss, sums, dh, dw, dv = torch.ops.b200rl.lm_linear_pg(h, w, rows, rows.long(), rows, None, None, None, rows,
                                                               'a2c', 1, 0.0, 0.0, 1, True, -0.01, 0.0, 0.5, False,
                                                               True, True)
        assert loss.shape == () and sums.shape == (3, ) and dh.numel() == 0 and dw.shape == w.shape
        assert dv.shape == (300, ) and dv.dtype == torch.float32


def test_every_language_model_function_traces():
    """every public function of the language-model losses -- the hidden-state module's and the reference's LM names --
    is compiled with fullgraph=True by this file or by tests/test_compile_lm.py, so a new one cannot slip in untraced"""
    from di_engine_b200.rl_utils import lm_linear
    public = [n for n in lm_linear.__all__ if not (isinstance(getattr(R, n), type) and issubclass(getattr(R, n), tuple))]
    public += list(R.LM_HOT_PATH_FUNCTIONS)
    traced = set(TRACED) | {v[1] for v in test_compile_lm.LOSSES.values()} | set(ALSO_TRACED)
    assert len(public) == 10 and not set(public) - traced, set(public) - traced


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
DEV = 'cuda'


@contextlib.contextmanager
def _chunks(V, dtype, lazy=True):
    """128-row chunks (300 rows: 128, 128, 44), and the monitors kept on the device: a python float leaves an inductor
    graph through a CPU kernel, which needs a host C++ toolchain with OpenMP"""
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(ops, 'LM_CHUNK_BYTES', 128 * V * torch.tensor([], dtype=dtype).element_size())
        mp.setattr(R.ppo, 'LAZY_INFO', lazy)
        yield


def _no_donated_buffers():
    """a second backward through a compiled graph (retain_graph) needs the saved intermediates kept: inductor otherwise
    donates their buffers to the first backward, and says so at the second"""
    import torch._functorch.config
    return torch._functorch.config.patch(donated_buffer=False)


def _gpu_data(kind, dtype, V, B=4, S=75, D=64, seed=0):
    if kind in ('grpo', 'rloo', 'logp'):
        d = tl.gpu_case('rloo' if kind == 'rloo' else 'grpo', dtype, B, S, D, V, seed=seed)
    else:
        d = tp.gpu_case(dtype, B, S, D, V, seed=seed)
    d['g'] = torch.randn(B, S, device=DEV)
    return d


def _leaves(kind, d):
    d = dict(d, hidden=d['hidden'].detach().clone().requires_grad_(True),
             lm_weight=d['lm_weight'].detach().clone().requires_grad_(True))
    leaves = [d['hidden'], d['lm_weight']]
    if kind == 'a2c':
        d['value'] = d['value'].detach().clone().requires_grad_(True)
        leaves.append(d['value'])
    return d, leaves


def _results(fn, kind, d, g_scale=1.0, twice=False, mark=None):
    """the call's outputs, then the gradients for ``g_scale * total``, then (``twice``) those of a second backward of
    ``-0.37 * total`` through the same graph; ``mark(d)`` marks dynamic dimensions on the leaves this call makes"""
    d, leaves = _leaves(kind, d)
    if mark is not None:
        mark(d)
    out, total = fn(kind, d)
    res = [x.detach().clone() for x in torch.utils._pytree.tree_leaves(out) if isinstance(x, torch.Tensor)]
    res += [g.clone() for g in torch.autograd.grad(g_scale * total, leaves, retain_graph=twice)]
    if twice:
        res += list(torch.autograd.grad(-0.37 * total, leaves))
    return res


def _same(got, want, what):
    assert len(got) == len(want), what
    for i, (a, b) in enumerate(zip(got, want)):
        assert a.dtype == b.dtype and a.shape == b.shape, (what, i)
        assert torch.equal(a, b) or (a.is_floating_point() and torch.equal(a.isnan(), b.isnan()) and
                                     torch.equal(a[~a.isnan()], b[~b.isnan()])), (what, i)


@pytest.mark.gpu
@pytest.mark.parametrize('kind', KINDS)
@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16], ids=['f32', 'bf16'])
def test_inductor_bit_identical_to_eager_over_several_chunks(kind, dtype):
    """unit, 0.5 and -2 upstream gradients, and a second backward with retain_graph: eager scales in place and recomputes
    on the second backward; the compiled call scales out of place and rescales the saved unit gradient"""
    V = 32771
    torch._dynamo.reset()
    f = torch.compile(_call, fullgraph=True)
    with _chunks(V, dtype), _no_donated_buffers():
        d = _gpu_data(kind, dtype, V)
        for g_scale, twice in ((1.0, False), (0.5, True), (-2.0, False)):
            got = _results(f, kind, d, g_scale, twice)
            want = _results(_call, kind, d, g_scale, twice)
            _same(got, want, (kind, dtype, g_scale))


def _fp64(kind, d):
    """the float64 reference of the test suites: d hidden and d lm_weight (and d value) of ``total``"""
    if kind in ('grpo', 'rloo'):
        return tl.fp64(kind, d)[3:]
    if kind == 'logp':
        h = d['hidden'].double().requires_grad_(True)
        w = d['lm_weight'].double().requires_grad_(True)
        (tl.go.logp64(h @ w.t(), d['action']) * d['g'].double()).sum().backward()
        return h.grad, w.grad
    return tp.fp64(kind, d, (None, 'k3', True))[1:4 if kind == 'a2c' else 3]


def _composition(kind, d):
    """F.linear + the library's logit losses: d hidden, d lm_weight (and d value), the yardstick of the bf16 rule"""
    if kind in ('grpo', 'rloo'):
        return tl.composition(kind, d)[3:]
    if kind == 'logp':
        h = d['hidden'].detach().clone().requires_grad_(True)
        w = d['lm_weight'].detach().clone().requires_grad_(True)
        (R.efficient_method(F.linear(h, w), d['action']) * d['g']).sum().backward()
        return h.grad, w.grad
    return tp.composition(kind, d, (None, 'k3', True))[1:4 if kind == 'a2c' else 3]


@pytest.mark.gpu
@pytest.mark.parametrize('kind', ('grpo', 'rloo', 'ppo', 'a2c', 'logp'))
@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16], ids=['f32', 'bf16'])
def test_compiled_gradients_under_upstream_not_one_and_second_backward_match_fp64(kind, dtype):
    """g = 0.5 on the first backward and -0.37 on a second one through the same graph: each gradient / g against the
    float64 reference, by the rules of tests/test_lm_linear.py (fp32: 1e-5 of the largest entry; bf16: twice the error
    of F.linear + the logit loss)"""
    V = 1003
    torch._dynamo.reset()
    f = torch.compile(_call, fullgraph=True)
    with _chunks(V, dtype), _no_donated_buffers():
        d = _gpu_data(kind, dtype, V)
        res = _results(f, kind, d, 0.5, twice=True)
        want = _fp64(kind, d)
        comp = _composition(kind, d)
    n = len(want)
    grads1, grads2 = res[-2 * n:-n], res[-n:]
    bf16 = dtype == torch.bfloat16
    for k in range(n):
        if want[k] is None:
            continue
        tl.check_tensor(grads1[k].double() / 0.5, comp[k], want[k], bf16)
        tl.check_tensor(grads2[k].double() / -0.37, comp[k], want[k], bf16)


@pytest.mark.gpu
@pytest.mark.parametrize('name', NEW_OPS)
def test_opcheck(name):
    if name == 'lm_linear_scale_out':
        for dtype in (torch.float32, torch.bfloat16):
            for n in (1, 7, 4099, 1 << 16):
                x = torch.randn(n, device=DEV).to(dtype)
                for g in (1.0, 0.37, -2.0):
                    gt = torch.tensor([g], device=DEV)
                    torch.library.opcheck(torch.ops.b200rl.lm_linear_scale_out, (gt, x))
                    want = x.clone()
                    ops.lm_scale_(ops.logit_dtype(want), gt.data_ptr(), want)  # eager's in-place scale
                    got = torch.ops.b200rl.lm_linear_scale_out(gt, x)
                    assert torch.equal(got.view(torch.int16 if dtype == torch.bfloat16 else torch.int32),
                                       want.view(torch.int16 if dtype == torch.bfloat16 else torch.int32)), (dtype, n, g)
            # a strided view: scaled as its values, into a contiguous tensor of its shape
            x = torch.randn(64, 130, device=DEV).to(dtype)[:, 1:128:3]
            gt = torch.tensor([0.37], device=DEV)
            torch.library.opcheck(torch.ops.b200rl.lm_linear_scale_out, (gt, x))
            got = torch.ops.b200rl.lm_linear_scale_out(gt, x)
            assert got.is_contiguous() and torch.equal(got, (x.float() * 0.37).to(dtype))
        return
    kind = {'lm_linear_loss': 'grpo', 'lm_linear_pg': 'a2c', 'lm_logp': 'logp', 'lm_logp_bwd': 'logp'}[name]
    mode, calls = _recording()
    with _chunks(1031, torch.float32), pytest.MonkeyPatch.context() as mp:
        d, leaves = _leaves(kind, _gpu_data(kind, torch.float32, 1031, seed=5))
        mp.setattr(torch.compiler, 'is_compiling', lambda: True)  # the traced path, run eagerly
        with mode:
            _, total = _call(kind, d)
            total.backward()
    found = [(op, a, k) for op, a, k in calls if op._opname == name]
    assert found, [op._opname for op, _, _ in calls]
    op, a, k = found[0]
    if name.endswith('_bwd'):  # a backward op is not differentiated again
        a, k = torch.utils._pytree.tree_map_only(torch.Tensor, lambda x: x.detach(), (a, k))
    with _chunks(1031, torch.float32):
        torch.library.opcheck(op, a, k)


@pytest.mark.gpu
@pytest.mark.parametrize('kind', ('grpo', 'rloo', 'ppo', 'a2c', 'logp'))
def test_dynamic_batch_and_length_do_not_recompile(kind):
    from torch._dynamo.utils import counters
    torch._dynamo.reset()
    counters.clear()
    f = torch.compile(_call, fullgraph=True)
    V = 1031
    with _chunks(V, torch.bfloat16):
        for B, S in ((4, 75), (6, 41), (8, 97)):
            d = _gpu_data(kind, torch.bfloat16, V, B=B, S=S, seed=S)

            def mark(e, B=B, S=S):
                for t in e.values():
                    if isinstance(t, torch.Tensor) and t.dim() >= 2 and t.shape[:2] == (B, S):
                        torch._dynamo.mark_dynamic(t, 0)
                        torch._dynamo.mark_dynamic(t, 1)
                    elif isinstance(t, torch.Tensor) and t.shape == (B, ):
                        torch._dynamo.mark_dynamic(t, 0)
                    elif isinstance(t, torch.Tensor) and t.shape == (2, B // 2):  # RLOO's reward (K, B / K)
                        torch._dynamo.mark_dynamic(t, 1)

            _same(_results(f, kind, d, mark=mark), _results(_call, kind, d), (kind, B, S))
    assert counters['stats']['unique_graphs'] == 1, dict(counters['stats'])


@pytest.mark.gpu
@pytest.mark.parametrize('kind', ('grpo', 'ppo', 'a2c'))
def test_reduce_overhead_replays_bit_identical_to_eager(kind):
    torch._dynamo.reset()
    f = torch.compile(_call, mode='reduce-overhead', fullgraph=True)
    V = 4099
    with _chunks(V, torch.bfloat16):
        for step in range(8):  # 2 warm-up / record calls, then replays
            d = _gpu_data(kind, torch.bfloat16, V, seed=step)
            _same(_results(f, kind, d), _results(_call, kind, d), (kind, step))


def _block(D, seed):
    torch.manual_seed(seed)
    return torch.nn.Sequential(torch.nn.Linear(D, D), torch.nn.Tanh()).to(DEV)


@pytest.mark.gpu
@pytest.mark.parametrize('kind', ('grpo', 'ppo', 'logp_no_grad'))
def test_learner_step_with_model_compiles_without_graph_break(kind):
    """a small Linear + tanh block in front of the loss; PPO adds ppo_value_error on a value head"""
    V, D = 1031, 64
    block = _block(D, 0)
    vhead = torch.nn.Linear(D, 1).to(DEV)
    d = _gpu_data('logp' if kind == 'logp_no_grad' else kind, torch.float32, V, D=D)
    w = d['lm_weight'].detach().clone().requires_grad_(True)

    def step(x):
        h = block(x)
        if kind == 'grpo':
            loss, info = R.grpo_policy_error_linear(R.grpo_linear_data(h, w, d['logp_old'], d['logp_ref'], d['action'],
                                                                       d['adv'], d['weight']))
            return loss, info.approx_kl
        if kind == 'ppo':
            out, info = R.ppo_policy_error_linear(R.ppo_policy_linear_data(h, w, d['logp_old'], d['action'], d['adv'],
                                                                           d['weight'], d['logp_pretrained']),
                                                  entropy_weight=0.01, kl_weight=0.1)
            v = R.ppo_value_error(R.ppo_value_data(vhead(h).squeeze(-1), d['value'], d['return_'], d['weight']), 0.2)
            return out.loss + 0.5 * v, info.clipfrac
        with torch.no_grad():
            return R.token_logp_linear(h, w, d['action']), None

    with _chunks(V, torch.float32):
        torch._dynamo.reset()
        explain = torch._dynamo.explain(step)(d['hidden'])
        assert explain.graph_break_count == 0, explain.break_reasons
        torch._dynamo.reset()
        res = []
        for fn in (step, torch.compile(step, backend='aot_eager', fullgraph=True)):
            for p in list(block.parameters()) + [w] + list(vhead.parameters()):
                p.grad = None
            loss, _ = fn(d['hidden'])
            if loss.requires_grad:
                loss.backward()
            res.append([loss.detach().clone()] + [p.grad.clone() for p in list(block.parameters()) + [w]
                                                  if p.grad is not None])
    _same(res[1], res[0], kind)


@pytest.mark.gpu
@pytest.mark.parametrize('kind', ('grpo', 'a2c'))
def test_peak_memory_bf16_no_higher_than_eager(kind):
    """bf16, D = 1024, V = 32 768, 8 x 1024 tokens: the compiled forward + backward peaks no higher than eager's (the
    out-of-place dW copy coexists with the saved one only after the forward's accumulator is gone)"""
    B, S, D, V = 8, 1024, 1024, 32768
    torch._dynamo.reset()
    f = torch.compile(_call, fullgraph=True)
    peaks = {}
    with _chunks(V, torch.bfloat16):
        monkey = pytest.MonkeyPatch()
        monkey.setattr(ops, 'LM_CHUNK_BYTES', 1 << 30)
        try:
            for mode, fn in (('warm', f), ('eager', _call), ('compiled', f)):
                d = _gpu_data(kind, torch.bfloat16, V, B=B, S=S, D=D)
                d, leaves = _leaves(kind, d)
                torch.cuda.synchronize()
                base = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
                grads = torch.autograd.grad(fn(kind, d)[1], leaves)
                torch.cuda.synchronize()
                peaks[mode] = torch.cuda.max_memory_allocated() - base
                del grads, d, leaves
        finally:
            monkey.undo()
    assert peaks['compiled'] <= peaks['eager'] + (8 << 20), peaks
