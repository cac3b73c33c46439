"""ppo_policy_error / ppo_error on language-model token rows (csrc/vocab.cu): dispatch, marshalling, errors and the float64
restatement against the reference's fixtures (CPU); the kernel against the fixtures, the restatement and the reference run
on the same CUDA tensors, the expected-gradient record, the old path, sizes up to (16, 1024, 32768) and (4, 128, 152064),
and the reference's own test_ppo_rlhf.py (GPU)."""
import contextlib
import inspect
import os

import numpy as np
import pytest
import torch

import di_engine_b200 as b2
from di_engine_b200 import ops
from tests import ppo_lm_oracle as po
from tests.test_grpo_rloo import _RecordingLib

R = b2.rl_utils
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'ppo_lm')
BF16_TOL = 2e-2  # the reference rounds every step to bf16 on bf16 logits (as test_grpo_rloo.py)
BF16_CLIPFRAC_TOL = 0.1


def gold(name):
    return dict(np.load(os.path.join(GOLD, name + '.npz')))


def close(got, want, tol):
    """|got - want| <= tol + tol * |want| (the project's bar)"""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    np.testing.assert_allclose(got, want, rtol=tol, atol=tol, equal_nan=True)


def close_grad(got, want, tol, bf16=False):
    """a gradient tensor against another, entry by entry within tol * (the wanted tensor's largest entry), plus the bf16
    rounding 2^-8 * |want| where the gradient is written in bf16 (`bf16`); in chunks, on the device of `got`"""
    got = torch.as_tensor(got).reshape(-1)
    want = torch.as_tensor(want).reshape(-1).to(got.device)
    scale = float(want.abs().max())
    if tol >= BF16_TOL:  # against the reference on bf16 logits: test_grpo_rloo.py's bar, scaled by max(1, largest entry)
        scale = max(scale, 1.0)
    for i in range(0, got.numel(), 1 << 24):
        g, w = got[i:i + (1 << 24)].double(), want[i:i + (1 << 24)].double()
        bound = tol * scale + (2.0 ** -8 * w.abs() if bf16 else 0.0)
        bad = ~((g - w).abs() <= bound)
        assert not bad.any(), 'entry %d: got %r want %r (scale %r), %d entries off' % (
            i + int(bad.nonzero()[0]), float(g[bad][0]), float(w[bad][0]), scale, int(bad.sum()))


def reference():
    from oracle import ref_loader
    if not ref_loader.available():
        pytest.skip('reference not importable here')
    return ref_loader.load()


def policy_call(d, dual_clip=None, kl_type='k1', entropy_bonus=True, clip=po.CLIP):
    data = R.ppo_policy_data(d['logit_new'], d['logit_old'], d['action'], d['adv'], d['weight'], d['logit_pretrained'])
    return R.ppo_policy_error(data, clip_ratio=clip, dual_clip=dual_clip, entropy_bonus=entropy_bonus, kl_type=kl_type)


def mixed(loss, has_kl, entropy_bonus, mix=po.MIX):
    total = mix[0] * loss.policy_loss
    if entropy_bonus:
        total = total + mix[1] * loss.entropy_loss
    if has_kl:
        total = total + mix[2] * loss.kl_div
    return total


def run_ours(d, dual_clip=None, kl_type='k1', entropy_bonus=True, mix=po.MIX, clip=po.CLIP):
    d = dict(d, logit_new=d['logit_new'].detach().clone().requires_grad_(True))
    loss, info = policy_call(d, dual_clip, kl_type, entropy_bonus, clip)
    mixed(loss, d['logit_pretrained'] is not None, entropy_bonus, mix).backward()
    vals = {'policy': loss.policy_loss.item(), 'entropy': float(loss.entropy_loss), 'kl': loss.kl_div.item(),
            'approx_kl': info.approx_kl, 'clipfrac': info.clipfrac}
    return vals, d['logit_new'].grad


# ----------------------------------------------------------------------------------------------------------------
# CPU: dispatch and marshalling against the ctypes prototypes, errors, the restatement against the reference
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


def lm_inputs(dtype, V, kl=True, B=2, S=3):
    return po.make_inputs(B, S, V, dtype, 'frac', kl, 0, 1.0, False)


@pytest.mark.parametrize('dtype,V', [(torch.bfloat16, 7), (torch.bfloat16, 1000), (torch.float32, 1024),
                                     (torch.float32, 1030)])
@pytest.mark.parametrize('kl', [False, True])
@pytest.mark.parametrize('entropy_bonus', [False, True])
def test_language_model_calls_marshal_into_the_vocab_entry_points(dry, dtype, V, kl, entropy_bonus):
    d = lm_inputs(dtype, V, kl)
    d['logit_new'].requires_grad_(True)
    loss, info = policy_call(d, entropy_bonus=entropy_bonus)
    assert isinstance(info.approx_kl, float) and isinstance(info.clipfrac, float)
    if not entropy_bonus:
        assert loss.entropy_loss.device.type == 'cpu' and not loss.entropy_loss.requires_grad
    mixed(loss, kl, entropy_bonus).backward()
    assert d['logit_new'].grad.dtype == dtype and d['logit_new'].grad.shape == d['logit_new'].shape
    assert dry.calls == ['b200rl_ppo_lm_fwd_grad', 'b200rl_ppo_lm_bwd']


def test_ppo_error_runs_the_policy_part_on_the_vocab_kernel(dry):
    d = lm_inputs(torch.bfloat16, 50)
    d['logit_new'].requires_grad_(True)
    v = torch.randn(2, 3, requires_grad=True)
    data = R.ppo_data(d['logit_new'], d['logit_old'], d['action'], v, v.detach() + 0.1, d['adv'], torch.randn(2, 3),
                      d['weight'], d['logit_pretrained'])
    loss, info = R.ppo_error(data)
    (loss.policy_loss + 0.5 * loss.value_loss - 0.01 * loss.entropy_loss + 0.1 * loss.kl_div).backward()
    assert dry.calls == ['b200rl_ppo_lm_fwd_grad', 'b200rl_ppo_value_fwd', 'b200rl_scale', 'b200rl_ppo_lm_bwd'] or \
        dry.calls == ['b200rl_ppo_lm_fwd_grad', 'b200rl_ppo_value_fwd', 'b200rl_ppo_lm_bwd', 'b200rl_scale']
    assert d['logit_new'].grad is not None and v.grad is not None


def test_record_kinds_are_the_existing_ones(dry):
    d = lm_inputs(torch.bfloat16, 9)
    d['logit_new'].requires_grad_(True)
    policy_call(d)
    v = torch.zeros(2, 3)
    R.ppo_error(R.ppo_data(d['logit_new'], d['logit_old'], d['action'], v, v, d['adv'], v, None, None))
    assert sorted(k for (_, k) in ops._HINT) == ['policy', 'ppo']


def test_lazy_info_returns_device_tensors(dry, monkeypatch):
    monkeypatch.setattr(R.ppo, 'LAZY_INFO', True)
    _, info = policy_call(lm_inputs(torch.bfloat16, 9))
    assert isinstance(info.approx_kl, torch.Tensor) and isinstance(info.clipfrac, torch.Tensor)


def test_weight_and_adv_of_any_dtype_are_read_as_fp32(dry):
    d = lm_inputs(torch.bfloat16, 9)
    d['weight'] = (d['weight'] > 0.5)
    d['adv'] = d['adv'].double()
    policy_call(d)
    assert dry.calls == ['b200rl_ppo_lm_fwd_grad']


@pytest.mark.parametrize('case', ['fp32_small_V', 'multi_agent', 'happo', 'adv_norm'])
def test_other_calls_keep_the_ppo_kernels(dry, case):
    if case == 'fp32_small_V':
        d = lm_inputs(torch.float32, 1023)
        policy_call(d)
        assert dry.calls == ['b200rl_ppo_fwd']
        return
    B, A, N = 4, 2, 1100
    x = torch.randn(B, A, N) if case == 'multi_agent' else torch.randn(B, N)
    act = torch.randint(0, N, x.shape[:-1])
    z = torch.zeros(B)
    if case == 'multi_agent':
        R.ppo_policy_error(R.ppo_policy_data(x, x + 0.1, act, torch.randn(B), None, None))
    elif case == 'happo':
        R.happo_policy_error(R.happo_policy_data(x, x + 0.1, act, torch.randn(B), None, torch.rand(B, 1)))
    else:
        R.ppo_error_adv_norm(R.ppo_data(x, x + 0.1, act, z, z, torch.randn(B), z, None, None))
    assert [c for c in dry.calls if c.startswith('b200rl_ppo')] == ['b200rl_ppo_fwd']


@pytest.mark.parametrize('case', ['multi_agent', 'happo', 'happo_policy', 'adv_norm', 'gae_ppo'])
def test_bf16_outside_the_language_model_shapes_raises(dry, case):
    B, A, N = 4, 2, 16
    x = (torch.randn(B, A, N) if case == 'multi_agent' else torch.randn(B, N)).bfloat16()
    act = torch.randint(0, N, x.shape[:-1])
    z = torch.zeros(B)
    with pytest.raises(TypeError) as e:
        if case == 'multi_agent':
            R.ppo_policy_error(R.ppo_policy_data(x, x, act, torch.randn(B), None, None))
        elif case == 'happo':
            R.happo_error(R.happo_data(x, x, act, z, z, torch.randn(B), z, None, torch.rand(B, 1)))
        elif case == 'happo_policy':
            R.happo_policy_error(R.happo_policy_data(x, x, act, torch.randn(B), None, torch.rand(B, 1)))
        elif case == 'adv_norm':
            R.ppo_error_adv_norm(R.ppo_data(x, x, act, z, z, torch.randn(B), z, None, None))
        else:
            T, Bs = 3, 4
            xs = torch.randn(T, Bs, N).bfloat16()
            zt = torch.zeros(T, Bs)
            R.gae_ppo_error(R.gae_data(zt, zt, zt, zt, zt),
                            R.ppo_data(xs, xs, torch.randint(0, N, (T, Bs)), zt, zt, None, zt, None, None))
    if case != 'gae_ppo':
        assert '(B, S, V) against (B, S)' in str(e.value)


def test_mixed_logit_dtypes_raise(dry):
    d = lm_inputs(torch.bfloat16, 9)
    d['logit_old'] = d['logit_old'].float()
    with pytest.raises(TypeError, match='share a dtype'):
        policy_call(d)


@pytest.mark.parametrize('name', sorted(po.CASES))
def test_restatement_matches_the_reference_fixtures(name):
    """the float64 restatement on the fixture's inputs against the reference's outputs: 1e-5 on fp32 inputs; on bf16 the
    reference rounds each step to bf16, so the bar there is bf16's"""
    d = po.make_case(name)
    g = gold(name)
    np.testing.assert_allclose(g['checksum'], po.checksum(d), rtol=1e-12)
    dual, kl_type, ent = po.case_args(name)
    want = po.run64(d, dual_clip=dual, kl_type=kl_type, entropy_bonus=ent)
    bf16 = po.CASES[name][0] == torch.bfloat16
    tol = BF16_TOL if bf16 else 1e-5
    for k in ('policy', 'entropy', 'kl', 'approx_kl'):
        close(g[k], want[k], tol)
    close(g['clipfrac'], want['clipfrac'], BF16_CLIPFRAC_TOL if bf16 else 1e-5)
    grad = want['grad'].reshape(-1)
    if 'grad' in g:
        close_grad(g['grad'], grad, tol)
    else:
        close_grad(g['grad_sample'], grad[g['grad_index']], tol)


def test_restatement_matches_the_live_reference():
    from tests.golden.make_ppo_lm_golden import reference_call
    ref = reference()
    for name in ('f32_v1003_mask_dc_k2', 'f32_v32771_frac_k3_inf'):
        d = po.make_case(name)
        dual, kl_type, ent = po.case_args(name)
        pol, e, kl, akl, cf, grad = reference_call(ref, d, dual, kl_type, ent)
        want = po.run64(d, dual_clip=dual, kl_type=kl_type, entropy_bonus=ent)
        for got, k in ((pol, 'policy'), (e, 'entropy'), (kl, 'kl'), (akl, 'approx_kl'), (cf, 'clipfrac')):
            close(got, want[k], 1e-5)
        close_grad(grad, want['grad'], 1e-5)


def test_signatures_and_namedtuples_match_the_reference():
    ref = reference()
    for name in ('ppo_policy_error', 'ppo_error'):
        po_, pt = inspect.signature(getattr(R, name)).parameters, inspect.signature(getattr(ref, name)).parameters
        assert list(po_) == list(pt), name
        assert all(po_[k].default == pt[k].default for k in po_), name
    for name in ('ppo_policy_data', 'ppo_policy_loss', 'ppo_data', 'ppo_loss', 'ppo_info'):
        assert getattr(R, name)._fields == getattr(ref, name)._fields, name


# ----------------------------------------------------------------------------------------------------------------
# GPU
# ----------------------------------------------------------------------------------------------------------------
DEV = 'cuda:0'


@pytest.fixture
def every_vocab(monkeypatch):
    """fp32 calls below LM_MIN_VOCAB take the vocabulary kernel too, so that fp32 V = 1000 / 1003 test it"""
    monkeypatch.setattr(R.ppo, 'LM_MIN_VOCAB', 1)


def to_dev(d):
    return {k: (v.to(DEV) if isinstance(v, torch.Tensor) else v) for k, v in d.items()}


def check_against(vals, grad, want, tol, clipfrac_tol=None, grad_index=None):
    for k in ('policy', 'entropy', 'kl', 'approx_kl'):
        close(vals[k], want[k], tol)
    close(vals['clipfrac'], want['clipfrac'], tol if clipfrac_tol is None else clipfrac_tol)
    g = grad.reshape(-1)
    if grad_index is not None:
        g = g[torch.as_tensor(grad_index, device=g.device)]
    close_grad(g, torch.as_tensor(want['grad']), tol, grad.dtype == torch.bfloat16)


@pytest.mark.gpu
@pytest.mark.parametrize('name', sorted(po.CASES))
def test_kernel_against_fixtures_restatement_and_reference(name, every_vocab):
    d = po.make_case(name, DEV)
    dual, kl_type, ent = po.case_args(name)
    bf16 = po.CASES[name][0] == torch.bfloat16
    vals, grad = run_ours(d, dual, kl_type, ent)
    # the float64 restatement on the same (for bf16: upcast) inputs: the project's bar
    want = po.run64(d, dual_clip=dual, kl_type=kl_type, entropy_bonus=ent)
    check_against(vals, grad, want, 1e-5)
    # the reference's outputs: the fixture (reference on the CPU) and the reference on the same CUDA tensors.  fp32: the
    # same bar; bf16: the reference rounds every step to bf16
    tol = BF16_TOL if bf16 else 1e-5
    cf_tol = BF16_CLIPFRAC_TOL if bf16 else None
    g = gold(name)
    gw = {k: g[k] for k in ('policy', 'entropy', 'kl', 'approx_kl', 'clipfrac')}
    check_against(vals, grad, dict(gw, grad=g.get('grad', g.get('grad_sample'))), tol, cf_tol, g.get('grad_index'))
    from tests.golden.make_ppo_lm_golden import reference_call
    from oracle import ref_loader
    if ref_loader.available():
        pol, e, kl, akl, cf, rgrad = reference_call(ref_loader.load(), d, dual, kl_type, ent)
        rw = {'policy': pol, 'entropy': e, 'kl': kl, 'approx_kl': akl, 'clipfrac': cf, 'grad': rgrad.float()}
        check_against(vals, grad, rw, tol, cf_tol)


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
@pytest.mark.parametrize('V', [1000, 1003, 1024, 32771])
@pytest.mark.parametrize('wkind', [None, 'mask', 'frac'])
@pytest.mark.parametrize('kl_type', [None, 'k1', 'k2', 'k3'])
@pytest.mark.parametrize('entropy_bonus', [False, True])
def test_parity_grid(dtype, V, wkind, kl_type, entropy_bonus, every_vocab):
    """every combination against the float64 restatement: the dual clip on for half of them (the advantages are half
    negative), -inf logits in the odd vocabularies, adv = 0 in one row of each"""
    B, S = (2, 3) if V > 10000 else (3, 7)
    seed = V + 10 * [None, 'mask', 'frac'].index(wkind) + 100 * [None, 'k1', 'k2', 'k3'].index(kl_type) + entropy_bonus
    d = po.make_inputs(B, S, V, dtype, wkind, kl_type is not None, seed, 2.0, V % 2 == 1, DEV)
    dual = 2.0 if seed % 2 else None
    vals, grad = run_ours(d, dual, kl_type or 'k1', entropy_bonus)
    want = po.run64(d, dual_clip=dual, kl_type=kl_type or 'k1', entropy_bonus=entropy_bonus)
    check_against(vals, grad, want, 1e-5)


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
def test_ratio_exactly_at_the_clip_bounds(dtype, every_vocab):
    """logit_old == logit_new: every ratio is exactly 1, and with clip_ratio = 0 that is 1 - clip and 1 + clip at once --
    min() ties, clamp() edges and the clipfrac comparisons all at the bound -- with positive, negative and zero
    advantages, against the float64 restatement and the reference"""
    d = po.make_inputs(3, 5, 1024, dtype, 'mask', True, 21, 1.0, False, DEV)
    d['logit_old'] = d['logit_new'].clone()
    d['adv'][1] = -d['adv'][1].abs()
    for clip, dual in ((0.0, None), (0.0, 2.0), (0.2, None)):
        vals, grad = run_ours(d, dual, 'k3', False, clip=clip)
        want = po.run64(d, clip=clip, dual_clip=dual, kl_type='k3', entropy_bonus=False)
        check_against(vals, grad, want, 1e-5)
        assert vals['clipfrac'] == 0.0 and vals['approx_kl'] == 0.0
        from tests.golden.make_ppo_lm_golden import reference_call
        from oracle import ref_loader
        if ref_loader.available():
            ref = ref_loader.load()
            x = dict(d, logit_new=d['logit_new'].clone())
            data = ref.ppo_policy_data(x['logit_new'].requires_grad_(True), d['logit_old'], d['action'], d['adv'],
                                       d['weight'], d['logit_pretrained'])
            loss, info = ref.ppo_policy_error(data, clip_ratio=clip, dual_clip=dual, entropy_bonus=False, kl_type='k3')
            close(vals['policy'], loss.policy_loss.item(), 1e-5 if dtype == torch.float32 else BF16_TOL)
            assert info.clipfrac == 0.0


def _record(kind='policy'):
    return ops.ppo_hint(torch.device(DEV), kind)


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
def test_expected_gradient_record(dtype):
    """the forward writes the gradient for the record's upstream gradients; a backward with others recomputes and is
    exact, and refreshes the record, so the next step with the same mix returns at once (a sentinel written into the
    forward's buffer survives: nothing recomputed it)"""
    d = po.make_inputs(4, 6, 4096, dtype, 'frac', True, 31, 2.0, False, DEV)
    mix = (1.0, -0.01, 0.1)
    want = po.run64(d, kl_type='k3', mix=mix)
    _record().copy_(torch.tensor([1.0, 0.0, -0.01, 0.0]))  # the record as a fresh process starts it
    for step in range(3):
        x = d['logit_new'].clone().requires_grad_(True)
        loss, _ = policy_call(dict(d, logit_new=x), kl_type='k3')
        fwd_grad, g_used = loss.policy_loss.grad_fn.spec
        hit = torch.equal(g_used.cpu(), torch.tensor([1.0, 0.0, -0.01, 0.1]))
        assert hit == (step > 0)
        if hit:
            fwd_grad.fill_(7.0)  # the verify launch returns at once: autograd hands this buffer on unchanged
        mixed(loss, True, True, mix).backward()
        if hit:
            assert bool((x.grad == 7.0).all())
        else:
            close_grad(x.grad, want['grad'], 1e-5, dtype == torch.bfloat16)
        assert torch.equal(_record().cpu(), torch.tensor([1.0, 0.0, -0.01, 0.1]))
    # and with no sentinel the verified gradient is exact
    x = d['logit_new'].clone().requires_grad_(True)
    loss, _ = policy_call(dict(d, logit_new=x), kl_type='k3')
    mixed(loss, True, True, mix).backward()
    close_grad(x.grad, want['grad'], 1e-5, dtype == torch.bfloat16)


@pytest.mark.gpu
@pytest.mark.parametrize('which', ['entropy', 'kl', 'policy_scaled', 'repeated'])
def test_backward_through_one_output(which):
    d = po.make_inputs(3, 5, 2048, torch.float32, 'mask', True, 41, 2.0, True, DEV)
    x = d['logit_new'].clone().requires_grad_(True)
    loss, _ = policy_call(dict(d, logit_new=x), kl_type='k2')
    if which == 'entropy':
        loss.entropy_loss.backward()
        mix = (0.0, 1.0, 0.0)
    elif which == 'kl':
        loss.kl_div.backward()
        mix = (0.0, 0.0, 1.0)
    elif which == 'policy_scaled':
        (2.5 * loss.policy_loss).backward()
        mix = (2.5, 0.0, 0.0)
    else:
        total = mixed(loss, True, True)
        total.backward(retain_graph=True)
        first = x.grad.clone()
        total.backward()
        close_grad(x.grad, 2 * first, 1e-6)
        mix = tuple(2 * m for m in po.MIX)
    want = po.run64(d, kl_type='k2', mix=mix)
    close_grad(x.grad, want['grad'], 1e-5)


@pytest.mark.gpu
@pytest.mark.parametrize('V', [1024, 4096])
@pytest.mark.parametrize('kl', [False, True])
def test_old_and_new_paths_agree(V, kl):
    """fp32 calls at V >= 1024 now run on csrc/vocab.cu; ops.PPOFunction (csrc/ppo.cu) still computes the same thing"""
    d = po.make_inputs(4, 8, V, torch.float32, 'frac', kl, 51 + V, 2.0, False, DEV)
    vals, grad = run_ours(d, 2.0, 'k3', True)
    rows = 32
    x = d['logit_new'].reshape(rows, V).clone().requires_grad_(True)
    z = torch.zeros(rows, device=DEV)
    pre = d['logit_pretrained'].reshape(rows, V).contiguous() if kl else None
    p, v, e, k, out = ops.PPOFunction.apply(
        x, z.clone().requires_grad_(True), d['logit_old'].reshape(rows, V).contiguous(), d['action'].reshape(-1), z,
        d['adv'].reshape(-1), z, d['weight'].reshape(-1).contiguous(), pre, rows, 1, V, po.CLIP, 0, 2.0, 3, 'policy')
    (p * po.MIX[0] + e * po.MIX[1] + (k * po.MIX[2] if kl else 0)).backward()
    for got, want in ((vals['policy'], p), (vals['entropy'], e), (vals['kl'], k), (vals['approx_kl'], out[4]),
                      (vals['clipfrac'], out[5])):
        close(got, want.item(), 1e-5)
    close_grad(grad, x.grad, 1e-5)


@pytest.mark.gpu
@pytest.mark.parametrize('shape,dtype', [((16, 1024, 32768), torch.float32), ((16, 1024, 32768), torch.bfloat16),
                                         ((4, 128, 152064), torch.bfloat16)])
def test_language_model_scale(shape, dtype):
    """against the reference on the same CUDA tensors, and the float64 restatement on 256 rows of them; the clip fraction
    may differ by one token whose ratio lies within rounding of a bound"""
    B, S, V = shape
    gen = torch.Generator(device=DEV).manual_seed(B + S + V)
    new = torch.randn(B, S, V, device=DEV, generator=gen, dtype=torch.float32) * 2
    d = {'logit_new': new.to(dtype),
         'logit_old': (new + 0.1 * torch.randn(B, S, V, device=DEV, generator=gen)).to(dtype),
         'logit_pretrained': (new + 0.2 * torch.randn(B, S, V, device=DEV, generator=gen)).to(dtype),
         'action': torch.randint(0, V, (B, S), device=DEV, generator=gen),
         'adv': torch.randn(B, S, device=DEV, generator=gen),
         'weight': (torch.rand(B, S, device=DEV, generator=gen) > 0.2).float()}
    del new
    bf16 = dtype == torch.bfloat16
    vals, grad = run_ours(d, None, 'k3', False)
    rows = B * S
    from tests.golden.make_ppo_lm_golden import reference_call
    from oracle import ref_loader
    if ref_loader.available():
        pol, e, kl, akl, cf, rgrad = reference_call(ref_loader.load(), d, None, 'k3', False)
        tol = BF16_TOL if bf16 else 1e-5
        for got, k in ((pol, 'policy'), (kl, 'kl'), (akl, 'approx_kl')):
            close(vals[k], got, tol)
        close(vals['clipfrac'], cf, BF16_CLIPFRAC_TOL if bf16 else 1.0 / rows + 1e-5)
        if not bf16:
            close_grad(grad, rgrad, 1e-5)
        del rgrad
    # 256 rows through the restatement: the means change with the subset, each row's gradient only by its 1 / M
    idx = torch.linspace(0, rows - 1, 256, device=DEV).long()
    sub = {k: d[k].reshape(rows, V)[idx].reshape(1, 256, V) for k in ('logit_new', 'logit_old', 'logit_pretrained')}
    sub.update({k: d[k].reshape(rows)[idx].reshape(1, 256) for k in ('action', 'adv', 'weight')})
    want = po.run64(sub, kl_type='k3', entropy_bonus=False)
    close_grad(grad.reshape(rows, V)[idx].double() * (rows / 256), want['grad'], 1e-5, bf16)


@pytest.mark.gpu
def test_host_tensors():
    d = po.make_case('bf16_v1003_frac_dc_k1')
    vals_h, grad_h = run_ours(d, 2.0, 'k1', True)
    vals_d, grad_d = run_ours(to_dev(d), 2.0, 'k1', True)
    assert grad_h.device.type == 'cpu'
    for k in vals_h:
        close(vals_h[k], vals_d[k], 0.0)
    assert torch.equal(grad_h, grad_d.cpu())


@pytest.mark.gpu
def test_ppo_error_at_language_model_shapes():
    d = po.make_inputs(2, 16, 2048, torch.bfloat16, 'mask', True, 61, 1.0, False, DEV)
    gen = torch.Generator().manual_seed(62)
    v = torch.randn(2, 16, generator=gen).to(DEV).requires_grad_(True)
    v_old, ret = (v.detach() + 0.1), torch.randn(2, 16, generator=gen).to(DEV)
    x = d['logit_new'].clone().requires_grad_(True)
    loss, info = R.ppo_error(R.ppo_data(x, d['logit_old'], d['action'], v, v_old, d['adv'], ret, d['weight'],
                                        d['logit_pretrained']), kl_type='k2')
    (loss.policy_loss + 0.5 * loss.value_loss - 0.01 * loss.entropy_loss + 0.1 * loss.kl_div).backward()
    want = po.run64(d, kl_type='k2', mix=(1.0, -0.01, 0.1))
    for k, got in (('policy', loss.policy_loss), ('entropy', loss.entropy_loss), ('kl', loss.kl_div)):
        close(got.item(), want[k], 1e-5)
    close_grad(x.grad, want['grad'], 1e-5, True)
    vv = v.detach().double().requires_grad_(True)
    w = d['weight'].double()
    vc = v_old.double() + (vv - v_old.double()).clamp(-po.CLIP, po.CLIP)
    vl = 0.5 * (torch.max((ret.double() - vv) ** 2, (ret.double() - vc) ** 2) * w).mean()
    (0.5 * vl).backward()
    close(loss.value_loss.item(), vl.item(), 1e-5)
    close_grad(v.grad, vv.grad, 1e-5)


# the reference's own tests (ding/rl_utils/tests/test_ppo_rlhf.py), run as written against this library on the GPU
@pytest.mark.gpu
@pytest.mark.parametrize('masked', [False, True])
def test_ported_policy_loss(masked, batch_size=4, seq_length=8, dictionary_num=1000):
    logit_new = torch.randn(batch_size, seq_length, dictionary_num, device=DEV).requires_grad_(True)
    logit_old = logit_new + torch.randn_like(logit_new) * 0.1
    logit_pretrained = logit_new + torch.randn_like(logit_new) * 0.1
    action = torch.randint(0, 10, (batch_size, seq_length), device=DEV)
    advantages = torch.randn(batch_size, seq_length, device=DEV)
    action_mask = None
    if masked:
        action_mask = torch.ones(batch_size, seq_length, device=DEV)
        action_mask[:, -2:] = 0
    data = R.ppo_policy_data(logit_new, logit_old, action, advantages, weight=action_mask,
                             logit_pretrained=logit_pretrained)
    loss, info = R.ppo_policy_error(data, clip_ratio=0.2, entropy_bonus=False)
    assert isinstance(loss.policy_loss, torch.Tensor)
    assert loss.policy_loss.shape == torch.Size([])
    assert not torch.isnan(loss.policy_loss)
    assert not torch.isinf(loss.policy_loss)
    assert logit_new.grad is None
    loss.policy_loss.backward()
    assert isinstance(logit_new.grad, torch.Tensor)
    assert all([np.isscalar(i) for i in info])


@pytest.mark.gpu
def test_ported_value_loss(batch_size=4, seq_length=8):
    values = torch.randn(batch_size, seq_length, device=DEV).requires_grad_(True)
    old_values = values + torch.randn_like(values) * 0.1
    returns = torch.randn(batch_size, seq_length, device=DEV)
    data = R.ppo_value_data(values, old_values, returns, weight=None)
    value_loss = R.ppo_value_error(data, clip_ratio=0.2, use_value_clip=True)
    assert isinstance(value_loss, torch.Tensor)
    assert value_loss.shape == torch.Size([])
    assert not torch.isnan(value_loss)
    assert not torch.isinf(value_loss)
    assert values.grad is None
    value_loss.backward()
    assert isinstance(values.grad, torch.Tensor)
