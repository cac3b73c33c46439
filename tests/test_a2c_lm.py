"""a2c_error on language-model token rows (csrc/vocab.cu): dispatch, marshalling, errors and the reference's fixtures
(CPU); the kernel against the fixtures, a float64 evaluation of oracle/rl_oracle.a2c_error and the reference run on the
same CUDA tensors, the expected-gradient record, the old path and sizes up to (16, 1024, 32768) and (4, 128, 152064)
(GPU)."""
import contextlib
import inspect
import os

import numpy as np
import pytest
import torch

import di_engine_b200 as b2
from di_engine_b200 import ops
from oracle import rl_oracle
from tests.golden import make_a2c_lm_golden as mk
from tests.test_grpo_rloo import _RecordingLib
from tests.test_ppo_lm import BF16_TOL, close, close_grad

R = b2.rl_utils
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'a2c_lm')
MIX = mk.MIX
RECORD_INIT = [1.0, 0.5, -0.01, 0.0]  # ops._HINT_INIT['a2c']


def gold(name):
    return dict(np.load(os.path.join(GOLD, name + '.npz')))


def reference():
    from oracle import ref_loader
    if not ref_loader.available():
        pytest.skip('reference not importable here')
    return ref_loader.load()


def run64(d, mix=MIX):
    """oracle/rl_oracle.a2c_error on float64 copies of d (bf16 logits upcast exactly) and d mix / d logit, d mix / d value"""
    x = d['logit'].detach().double().requires_grad_(True)
    v = d['value'].detach().double().requires_grad_(True)
    w = d['weight'].double() if d['weight'] is not None else None
    p, vl, e = rl_oracle.a2c_error(x, d['action'], v, d['adv'].double(), d['return_'].double(), w)
    (mix[0] * p + mix[1] * vl + mix[2] * e).backward()
    return {'policy': p.item(), 'value': vl.item(), 'entropy': e.item(), 'grad': x.grad, 'grad_value': v.grad}


def a2c_call(d, x, v):
    return R.a2c_error(R.a2c_data(x, d['action'], v, d['adv'], d['return_'], d['weight']))


def run_ours(d, mix=MIX):
    x = d['logit'].detach().clone().requires_grad_(True)
    v = d['value'].detach().clone().requires_grad_(True)
    loss = a2c_call(d, x, v)
    (mix[0] * loss.policy_loss + mix[1] * loss.value_loss + mix[2] * loss.entropy_loss).backward()
    vals = {'policy': loss.policy_loss.item(), 'value': loss.value_loss.item(), 'entropy': loss.entropy_loss.item()}
    return vals, x.grad, v.grad


def check_against(vals, grad, grad_value, want, tol, grad_index=None):
    for k in ('policy', 'value', 'entropy'):
        close(vals[k], want[k], tol)
    g = grad.reshape(-1)
    if grad_index is not None:
        g = g[torch.as_tensor(grad_index, device=g.device)]
    close_grad(g, torch.as_tensor(want['grad']), tol, grad.dtype == torch.bfloat16)
    close_grad(grad_value, torch.as_tensor(want['grad_value']), tol)


# ----------------------------------------------------------------------------------------------------------------
# CPU: dispatch and marshalling against the ctypes prototypes, errors, the fixtures against the reference
# ----------------------------------------------------------------------------------------------------------------
@pytest.fixture
def dry(monkeypatch):
    rec = _RecordingLib()
    monkeypatch.setattr(ops, 'lib', lambda: rec)
    monkeypatch.setattr(ops, 'require_cuda', lambda: None)
    monkeypatch.setattr(ops, 'compute_device', lambda *t: torch.device('cpu'))
    monkeypatch.setattr(ops, 'stream_ptr', lambda: 0)
    monkeypatch.setattr(torch.cuda, 'device', lambda d: contextlib.nullcontext())
    ops._WS.clear()
    ops._HINT.clear()
    yield rec
    ops._WS.clear()
    ops._HINT.clear()


def lm_inputs(dtype, V, wkind='frac', B=2, S=3):
    return mk.make_inputs(B, S, V, dtype, wkind, 0, 1.0, False, False)


@pytest.mark.parametrize('dtype,V,entry', [(torch.float32, 1023, 'b200rl_a2c_fwd_grad'),
                                           (torch.float32, 1024, 'b200rl_a2c_lm_fwd_grad'),
                                           (torch.float32, 4096, 'b200rl_a2c_lm_fwd_grad'),
                                           (torch.bfloat16, 7, 'b200rl_a2c_lm_fwd_grad'),
                                           (torch.bfloat16, 1000, 'b200rl_a2c_lm_fwd_grad')])
@pytest.mark.parametrize('wkind', [None, 'mask'])
def test_dispatch_and_marshalling(dry, dtype, V, entry, wkind):
    d = lm_inputs(dtype, V, wkind)
    x, v = d['logit'].clone().requires_grad_(True), d['value'].clone().requires_grad_(True)
    loss = a2c_call(d, x, v)
    (loss.policy_loss + 0.5 * loss.value_loss - 0.01 * loss.entropy_loss).backward()
    bwd = 'b200rl_a2c_fwd_grad' if entry == 'b200rl_a2c_fwd_grad' else 'b200rl_a2c_lm_bwd'
    assert dry.calls == [entry, bwd]
    assert x.grad.dtype == dtype and x.grad.shape == x.shape
    assert v.grad.dtype == torch.float32 and v.grad.shape == v.shape


def test_bf16_value_gets_a_bf16_gradient(dry):
    d = lm_inputs(torch.bfloat16, 9)
    x = d['logit'].clone().requires_grad_(True)
    v = d['value'].bfloat16().requires_grad_(True)
    loss = a2c_call(d, x, v)
    loss.value_loss.backward()
    assert v.grad.dtype == torch.bfloat16 and v.grad.shape == v.shape
    assert dry.calls == ['b200rl_a2c_lm_fwd_grad', 'b200rl_a2c_lm_bwd']


def test_operands_of_any_dtype_are_read_as_fp32(dry):
    d = lm_inputs(torch.bfloat16, 9)
    d['weight'] = d['weight'] > 0.5
    d['adv'], d['return_'] = d['adv'].double(), d['return_'].half()
    d['action'] = d['action'].int()
    a2c_call(d, d['logit'], d['value'])
    assert dry.calls == ['b200rl_a2c_lm_fwd_grad']


def test_no_gradient_wanted_passes_no_gradient_buffers(dry):
    d = lm_inputs(torch.float32, 2048)
    with torch.no_grad():
        loss = a2c_call(d, d['logit'], d['value'])
    assert dry.calls == ['b200rl_a2c_lm_fwd_grad'] and loss.policy_loss.grad_fn is None


def test_record_kind_is_the_existing_one(dry):
    d = lm_inputs(torch.bfloat16, 9)
    a2c_call(d, d['logit'].clone().requires_grad_(True), d['value'])
    assert sorted(k for (_, k) in ops._HINT) == ['a2c']


@pytest.mark.parametrize('name', ['action', 'value', 'adv', 'return_', 'weight'])
@pytest.mark.parametrize('dtype,V', [(torch.bfloat16, 9), (torch.float32, 1024)])
def test_operand_size_mismatch_raises_value_error(dry, name, dtype, V):
    d = lm_inputs(dtype, V)
    d[name] = torch.cat([d[name].reshape(-1), d[name].reshape(-1)[:1]])
    with pytest.raises(ValueError, match=name):
        a2c_call(d, d['logit'], d['value'])
    assert dry.calls == []


@pytest.mark.parametrize('dtype', [torch.float16, torch.float64])
@pytest.mark.parametrize('V', [9, 1024])
def test_fp16_and_fp64_logits_raise_type_error(dry, dtype, V):
    d = lm_inputs(torch.float32, V)
    with pytest.raises(TypeError):
        a2c_call(d, d['logit'].to(dtype), d['value'])
    assert dry.calls == []


@pytest.mark.parametrize('dtype', [torch.float16, torch.float64])
def test_value_outside_fp32_and_bf16_raises_type_error(dry, dtype):
    d = lm_inputs(torch.bfloat16, 9)
    with pytest.raises(TypeError, match='value'):
        a2c_call(d, d['logit'], d['value'].to(dtype))
    assert dry.calls == []


def test_logit_dtype_check_is_the_vocab_one(dry, monkeypatch):
    seen = []
    real = ops.logit_dtype
    monkeypatch.setattr(ops, 'logit_dtype', lambda *t: seen.append(t[0].dtype) or real(*t))
    d = lm_inputs(torch.bfloat16, 9)
    a2c_call(d, d['logit'], d['value'])
    assert seen == [torch.bfloat16]


@pytest.mark.parametrize('name', sorted(mk.CASES))
def test_fixtures_match_the_float64_evaluation(name):
    """the fixture (the reference on the CPU) against oracle/rl_oracle.a2c_error in float64 on the same inputs: 1e-5 on
    fp32 logits; on bf16 the reference rounds each step to bf16, so the bar there is bf16's"""
    d = mk.make_case(name)
    g = gold(name)
    np.testing.assert_allclose(g['checksum'], mk.checksum(d), rtol=1e-12)
    want = run64(d)
    tol = BF16_TOL if mk.CASES[name][0] == torch.bfloat16 else 1e-5
    for k in ('policy', 'value', 'entropy'):
        close(g[k], want[k], tol)
    close_grad(g['grad_value'], want['grad_value'], 1e-5)
    grad = want['grad'].reshape(-1)
    if 'grad' in g:
        close_grad(g['grad'], grad, tol)
    else:
        close_grad(g['grad_sample'], grad[g['grad_index']], tol)


@pytest.mark.parametrize('name', sorted(mk.CASES))
def test_fixtures_match_the_live_reference(name):
    ref = reference()
    d = mk.make_case(name)
    g = gold(name)
    pol, val, ent, grad, gv = mk.reference_call(ref, d)
    for got, k in ((pol, 'policy'), (val, 'value'), (ent, 'entropy')):
        close(got, g[k], 0.0)
    grad = grad.float().reshape(-1).numpy()
    np.testing.assert_array_equal(grad if 'grad' in g else grad[g['grad_index']], g.get('grad', g.get('grad_sample')))
    np.testing.assert_array_equal(gv.reshape(-1).numpy(), g['grad_value'])


def test_signature_and_namedtuples_match_the_reference():
    ref = reference()
    assert list(inspect.signature(R.a2c_error).parameters) == list(inspect.signature(ref.a2c_error).parameters)
    for name in ('a2c_data', 'a2c_loss'):
        assert getattr(R, name)._fields == getattr(ref, name)._fields, name


# ----------------------------------------------------------------------------------------------------------------
# GPU
# ----------------------------------------------------------------------------------------------------------------
DEV = 'cuda:0'


@pytest.fixture
def every_vocab(monkeypatch):
    """fp32 calls below LM_MIN_VOCAB take the vocabulary kernel too, so that fp32 V = 1003 tests it"""
    monkeypatch.setattr(R.ppo, 'LM_MIN_VOCAB', 1)


def _record():
    return ops.ppo_hint(torch.device(DEV), 'a2c')


@pytest.fixture
def fresh_record():
    _record().copy_(torch.tensor(RECORD_INIT))  # the record as a fresh process starts it
    yield
    _record().copy_(torch.tensor(RECORD_INIT))


@pytest.mark.gpu
@pytest.mark.parametrize('name', sorted(mk.CASES))
def test_kernel_against_fixtures_float64_and_reference(name, every_vocab, fresh_record):
    d = mk.make_case(name, DEV)
    bf16 = mk.CASES[name][0] == torch.bfloat16
    vals, grad, gv = run_ours(d)
    # float64 on the same (for bf16: upcast) inputs: the project's bar
    check_against(vals, grad, gv, run64(d), 1e-5)
    # the reference's outputs: the fixture (reference on the CPU) and the reference on the same CUDA tensors.  fp32: the
    # same bar; bf16: the reference rounds every step to bf16
    tol = BF16_TOL if bf16 else 1e-5
    g = gold(name)
    gw = {'policy': g['policy'], 'value': g['value'], 'entropy': g['entropy'], 'grad_value': g['grad_value'],
          'grad': g.get('grad', g.get('grad_sample'))}
    check_against(vals, grad, gv, gw, tol, g.get('grad_index'))
    from oracle import ref_loader
    if ref_loader.available():
        pol, val, ent, rgrad, rgv = mk.reference_call(ref_loader.load(), d)
        rw = {'policy': pol, 'value': val, 'entropy': ent, 'grad': rgrad.float(), 'grad_value': rgv}
        check_against(vals, grad, gv, rw, tol)


@pytest.mark.gpu
@pytest.mark.parametrize('dtype,V', [(torch.float32, 1003), (torch.float32, 1024), (torch.float32, 32771),
                                     (torch.bfloat16, 1000), (torch.bfloat16, 1003), (torch.bfloat16, 1024),
                                     (torch.bfloat16, 32771)])
@pytest.mark.parametrize('wkind', [None, 'mask', 'frac'])
@pytest.mark.parametrize('peaked', [False, True])
def test_parity_grid(dtype, V, wkind, peaked, every_vocab, fresh_record):
    """against the float64 evaluation: -inf logits in the odd vocabularies, adv = 0 in one row of each, peaked rows
    (H ~ 0, and lp ~ -60) in half"""
    B, S = (2, 3) if V > 10000 else (3, 7)
    seed = V + 10 * [None, 'mask', 'frac'].index(wkind) + 100 * peaked
    d = mk.make_inputs(B, S, V, dtype, wkind, seed, 2.0, V % 2 == 1, peaked, DEV)
    vals, grad, gv = run_ours(d)
    check_against(vals, grad, gv, run64(d), 1e-5)


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
def test_expected_gradient_record(dtype, fresh_record):
    """the forward writes both gradients for the record's upstream gradients: with the default mix the backward returns
    at once on the device (sentinels written into the forward's buffers survive); another mix recomputes exactly and
    refreshes the record, so the next step with it returns at once; a change of the value weight alone rewrites d / d
    value only (the forward's d / d logit, still exact, is kept) and is exact"""
    d = mk.make_inputs(4, 6, 4096, dtype, 'frac', 31, 2.0, True, True, DEV)
    # (mix, forward-written logit gradient kept, value gradient kept)
    steps = [(MIX, True, True), ((2.0, 0.5, 0.3), False, False), ((2.0, 0.5, 0.3), True, True),
             ((2.0, 0.25, 0.3), True, False), ((2.0, 0.25, 0.3), True, True), ((2.0, 0.25, -0.7), False, False)]
    for mix, keep_logit, keep_value in steps:
        want = run64(d, mix)
        x = d['logit'].clone().requires_grad_(True)
        v = d['value'].clone().requires_grad_(True)
        loss = a2c_call(d, x, v)
        fwd_grad, fwd_gv, _ = loss.policy_loss.grad_fn.spec
        fwd_grad.fill_(7.0)
        fwd_gv.fill_(7.0)
        (mix[0] * loss.policy_loss + mix[1] * loss.value_loss + mix[2] * loss.entropy_loss).backward()
        if keep_logit:
            assert bool((x.grad == 7.0).all())
        else:
            close_grad(x.grad, want['grad'], 1e-5, dtype == torch.bfloat16)
        if keep_value:
            assert bool((v.grad == 7.0).all())
        else:
            close_grad(v.grad, want['grad_value'], 1e-5)
        assert torch.equal(_record().cpu(), torch.tensor(list(mix) + [0.0]))
        # and with no sentinel the handed-on gradients are exact
        vals, grad, gv = run_ours(d, mix)
        check_against(vals, grad, gv, want, 1e-5)


@pytest.mark.gpu
@pytest.mark.parametrize('which', ['policy', 'value', 'entropy', 'policy_scaled', 'repeated'])
@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
def test_backward_through_one_output(which, dtype, fresh_record):
    d = mk.make_inputs(3, 5, 2048, dtype, 'mask', 41, 2.0, True, False, DEV)
    x = d['logit'].clone().requires_grad_(True)
    v = d['value'].clone().requires_grad_(True)
    loss = a2c_call(d, x, v)
    if which in ('policy', 'value', 'entropy'):
        getattr(loss, which + '_loss').backward()
        mix = tuple(float(k == which) for k in ('policy', 'value', 'entropy'))
    elif which == 'policy_scaled':
        (2.5 * loss.policy_loss).backward()
        mix = (2.5, 0.0, 0.0)
    else:
        total = MIX[0] * loss.policy_loss + MIX[1] * loss.value_loss + MIX[2] * loss.entropy_loss
        total.backward(retain_graph=True)
        first, first_v = x.grad.clone(), v.grad.clone()
        total.backward()
        close_grad(x.grad, 2 * first, 1e-6 if dtype == torch.float32 else 2.0 ** -8)
        close_grad(v.grad, 2 * first_v, 1e-6)
        mix = tuple(2 * m for m in MIX)
    want = run64(d, mix)
    close_grad(x.grad, want['grad'], 1e-5, dtype == torch.bfloat16)
    close_grad(v.grad, want['grad_value'], 1e-5)


@pytest.mark.gpu
def test_bf16_value_gets_a_bf16_gradient_on_the_device(fresh_record):
    d = mk.make_inputs(2, 8, 1024, torch.bfloat16, 'frac', 43, 1.0, False, False, DEV)
    d['value'] = d['value'].bfloat16()
    vals, grad, gv = run_ours(d)
    assert gv.dtype == torch.bfloat16
    want = run64(d)  # value upcast exactly
    for k in ('policy', 'value', 'entropy'):
        close(vals[k], want[k], 1e-5)
    close_grad(gv, want['grad_value'], 1e-5, True)
    close_grad(grad, want['grad'], 1e-5, True)


@pytest.mark.gpu
@pytest.mark.parametrize('wkind', [None, 'frac'])
def test_old_and_new_paths_agree(wkind, fresh_record):
    """fp32 calls at V >= 1024 now run on csrc/vocab.cu; ops.A2CFunction (csrc/heads.cu) still computes the same thing"""
    V = 1024
    d = mk.make_inputs(4, 8, V, torch.float32, wkind, 51, 2.0, False, True, DEV)
    vals, grad, gv = run_ours(d)
    rows = 32
    x = d['logit'].reshape(rows, V).clone().requires_grad_(True)
    v = d['value'].reshape(rows).clone().requires_grad_(True)
    w = d['weight'].reshape(rows).contiguous() if wkind else None
    p, vl, e = ops.A2CFunction.apply(x, v, d['action'].reshape(rows), d['adv'].reshape(rows),
                                     d['return_'].reshape(rows), w, rows, V)
    (MIX[0] * p + MIX[1] * vl + MIX[2] * e).backward()
    for got, want in ((vals['policy'], p), (vals['value'], vl), (vals['entropy'], e)):
        close(got, want.item(), 1e-5)
    close_grad(grad, x.grad, 1e-5)
    close_grad(gv.reshape(-1), v.grad, 1e-5)


@pytest.mark.gpu
@pytest.mark.parametrize('shape,dtype', [((16, 1024, 32768), torch.float32), ((16, 1024, 32768), torch.bfloat16),
                                         ((4, 128, 152064), torch.bfloat16)])
def test_language_model_scale(shape, dtype, fresh_record):
    """against the reference on the same CUDA tensors, and the float64 evaluation on 256 rows of them"""
    B, S, V = shape
    gen = torch.Generator(device=DEV).manual_seed(B + S + V)
    d = {'logit': (torch.randn(B, S, V, device=DEV, generator=gen) * 2).to(dtype),
         'action': torch.randint(0, V, (B, S), device=DEV, generator=gen),
         'value': torch.randn(B, S, device=DEV, generator=gen),
         'adv': torch.randn(B, S, device=DEV, generator=gen),
         'return_': torch.randn(B, S, device=DEV, generator=gen),
         'weight': (torch.rand(B, S, device=DEV, generator=gen) > 0.2).float()}
    bf16 = dtype == torch.bfloat16
    vals, grad, gv = run_ours(d)
    rows = B * S
    from oracle import ref_loader
    if ref_loader.available():
        pol, val, ent, rgrad, rgv = mk.reference_call(ref_loader.load(), d)
        tol = BF16_TOL if bf16 else 1e-5
        for got, k in ((pol, 'policy'), (val, 'value'), (ent, 'entropy')):
            close(vals[k], got, tol)
        close_grad(gv, rgv, 1e-5)
        if not bf16:
            close_grad(grad, rgrad, 1e-5)
        del rgrad
    # 256 rows through float64: the means change with the subset, each row's gradient only by its 1 / M
    idx = torch.linspace(0, rows - 1, 256, device=DEV).long()
    sub = {'logit': d['logit'].reshape(rows, V)[idx].reshape(1, 256, V)}
    sub.update({k: d[k].reshape(rows)[idx].reshape(1, 256) for k in ('action', 'value', 'adv', 'return_', 'weight')})
    want = run64(sub)
    close_grad(grad.reshape(rows, V)[idx].double() * (rows / 256), want['grad'].reshape(256, V), 1e-5, bf16)
    close_grad(gv.reshape(rows)[idx].double() * (rows / 256), want['grad_value'].reshape(256), 1e-5)


@pytest.mark.gpu
def test_host_tensors(fresh_record):
    d = mk.make_case('bf16_v1003_frac_peaked')
    vals_h, grad_h, gv_h = run_ours(d)
    vals_d, grad_d, gv_d = run_ours({k: (t.to(DEV) if isinstance(t, torch.Tensor) else t) for k, t in d.items()})
    assert grad_h.device.type == 'cpu' and gv_h.device.type == 'cpu'
    for k in vals_h:
        close(vals_h[k], vals_d[k], 0.0)
    assert torch.equal(grad_h, grad_d.cpu()) and torch.equal(gv_h, gv_d.cpu())


@pytest.mark.gpu
def test_deterministic_loss_sums(fresh_record):
    d = mk.make_inputs(8, 64, 4099, torch.bfloat16, 'frac', 71, 2.0, True, True, DEV)
    first = run_ours(d)
    for _ in range(2):
        again = run_ours(d)
        assert again[0] == first[0]
        assert torch.equal(again[1], first[1]) and torch.equal(again[2], first[2])
