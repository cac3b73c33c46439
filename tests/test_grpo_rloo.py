"""grpo_policy_error, rloo_policy_error and the per-token log-prob methods (csrc/vocab.cu): marshalling, errors, the
float64 restatement against the reference's fixtures (CPU); the kernels against fixtures, the float64 restatement and the
reference's own tests, on fp32 and bf16 logits up to (16, 1024, 32768) and V = 152 064 (GPU)."""
import contextlib
import inspect
import os
import sys

import numpy as np
import pytest
import torch

import di_engine_b200 as b2
from di_engine_b200 import _lib, ops
from tests import grpo_oracle as go

R = b2.rl_utils
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'grpo_rloo')
LM_MODULES = ('grpo', 'rloo', 'log_prob_utils')
# the reference rounds the ratio to bf16 on bf16 logits (8 bits of mantissa): a token whose ratio lies within that rounding
# of 1 -+ clip may count as clipped there and not in fp32 -- up to a few tokens of the fixtures' 32
BF16_CLIPFRAC_TOL = {torch.bfloat16: 0.1}


def gold(name):
    return dict(np.load(os.path.join(GOLD, name + '.npz')))


def close(got, want, tol):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    finite = np.abs(want[np.isfinite(want)])
    scale = max(1.0, float(finite.max())) if finite.size else 1.0
    np.testing.assert_allclose(got, want, rtol=tol, atol=tol * scale, equal_nan=True)


@contextlib.contextmanager
def live_reference():
    """ding.rl_utils.{grpo, rloo, log_prob_utils} of the unmodified reference (its tree, or the archive build() made from
    it, oracle/ref_lm.py); skips where neither exists"""
    from oracle import ref_lm
    if not ref_lm.available():
        pytest.skip('reference not importable here')
    with ref_lm.modules() as mods:
        yield mods


def close_grad(got, want, scale, bf16, tol=1e-5):
    """d loss / d logit_new, row by row on the device, against want = dlp[row] * (onehot - softmax): each entry within
    tol * scale[row] + rtol * |want| (rtol = tol on fp32, the bf16 rounding 2^-8 on bf16 logits).  scale is the size of
    the terms that make up the row's dlp (grpo_oracle.run64's 'scale'; the upstream gradient for the log-prob methods),
    not the gradient's largest entry, so the softmax term of every entry is checked at its own size, however small 1 / V
    makes it; NaN where both are NaN"""
    V = want.shape[-1]
    got, want = got.reshape(-1, V), want.reshape(-1, V)
    scale = scale.abs().to(want.device, torch.float64).reshape(-1, 1)
    rtol = 2.0 ** -8 if bf16 else tol
    for r0 in range(0, got.shape[0], 256):
        g, w = got[r0:r0 + 256].double().to(want.device), want[r0:r0 + 256].double()
        bound = tol * scale[r0:r0 + 256] + rtol * w.abs()
        bad = ~((g - w).abs() <= bound) & ~(torch.isnan(g) & torch.isnan(w))
        if bad.any():
            i = bad.nonzero()[0]
            row, col = r0 + int(i[0]), int(i[1])
            raise AssertionError('row %d col %d: got %r want %r (dlp %r), %d entries off' %
                                 (row, col, float(g[i[0], i[1]]), float(w[i[0], i[1]]), float(scale[row]),
                                  int(bad.sum())))


def want64(d):
    """the float64 restatement of case d and its d loss / d logit_new (B, S, V), on d's device"""
    want = go.run64(d)
    grad64 = torch.stack([go.grad_rows64(d['logit_new'][b], d['action'][b], want['dlp'][b])
                          for b in range(d['action'].shape[0])])
    return want, grad64


def ref_call(ref, kind, d):
    """the reference's own loss on the tensors of d (any device): loss, info, d loss / d logit_new"""
    x = d['logit_new'].detach().clone().requires_grad_(True)
    if kind == 'grpo':
        loss, info = ref['grpo'].grpo_policy_error(ref['grpo'].grpo_policy_data(
            x, d['logit_old'], d['logit_ref'], d['action'], d['adv'], d['weight']), clip_ratio=go.CLIP, beta=go.BETA)
    else:
        loss, info = ref['rloo'].rloo_policy_error(ref['rloo'].rloo_policy_data(
            x, d['logit_old'], d['action'], d['reward'], d['weight']), clip_ratio=go.CLIP)
    loss.backward()
    return loss.item(), info, x.grad


def call(kind, d, fn=None, **kw):
    fn = R.efficient_method if fn is None else fn
    if kind == 'grpo':
        data = R.grpo_policy_data(d['logit_new'], d['logit_old'], d['logit_ref'], d['action'], d['adv'], d['weight'])
        return R.grpo_policy_error(data, fn, **kw)
    data = R.rloo_policy_data(d['logit_new'], d['logit_old'], d['action'], d['reward'], d['weight'])
    return R.rloo_policy_error(data, fn, **kw)


# ----------------------------------------------------------------------------------------------------------------
# CPU: marshalling against the ctypes prototypes, errors, the restatement against the reference
# ----------------------------------------------------------------------------------------------------------------
class _RecordingLib:

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        proto = _lib.PROTOTYPES[name]

        def fn(*args):
            assert len(args) == len(proto), (name, len(args), len(proto))
            for a, ty in zip(args, proto):
                ty.from_param(a)
            self.calls.append(name)
            return 0

        if name == 'b200rl_workspace_bytes':
            return lambda: 1 << 20
        return fn


@pytest.fixture
def dry(monkeypatch):
    rec = _RecordingLib()
    monkeypatch.setattr(ops, 'lib', lambda: rec)
    monkeypatch.setattr(ops, 'require_cuda', lambda: None)
    monkeypatch.setattr(ops, 'compute_device', lambda *t: torch.device('cpu'))
    monkeypatch.setattr(ops, 'stream_ptr', lambda: 0)
    monkeypatch.setattr(torch.cuda, 'device', lambda d: contextlib.nullcontext())
    ops._WS.clear()
    yield rec
    ops._WS.clear()


@pytest.mark.parametrize('kind', ['grpo', 'rloo'])
@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
@pytest.mark.parametrize('weighted', [False, True])
def test_fused_call_marshals(dry, kind, dtype, weighted):
    d = go.make_case('grpo_f32_mask' if kind == 'grpo' else 'rloo_f32_k8_mask')
    for k in ('logit_new', 'logit_old', 'logit_ref'):
        if k in d:
            d[k] = d[k].to(dtype)
    if not weighted:
        d['weight'] = None
    d['logit_new'].requires_grad_(True)
    loss, info = call(kind, d)
    assert loss.shape == () and isinstance(info.approx_kl, float) and isinstance(info.clipfrac, float)
    loss.backward()
    assert d['logit_new'].grad.dtype == dtype and d['logit_new'].grad.shape == d['logit_new'].shape
    assert dry.calls == ['b200rl_%s_fwd_grad' % kind, 'b200rl_token_logp_bwd']


@pytest.mark.parametrize('method', ['naive_method', 'efficient_method', 'less_efficient_method'])
@pytest.mark.parametrize('shape', [(3, 5, 7), (5, 7)])
def test_log_prob_methods_marshal(dry, method, shape):
    x = torch.randn(*shape, requires_grad=True)
    idx = torch.randint(0, shape[-1], shape[:-1])
    lp = getattr(R, method)(x, idx)
    assert lp.shape == shape[:-1] and lp.dtype == torch.float32
    lp.sum().backward()
    assert dry.calls == ['b200rl_token_logp_fwd', 'b200rl_token_logp_bwd']


@pytest.mark.parametrize('kind', ['grpo', 'rloo'])
def test_custom_log_prob_fn_marshals(dry, kind):
    d = go.make_case('grpo_f32_v33' if kind == 'grpo' else 'rloo_f32_k2_zero_row')
    d['logit_new'].requires_grad_(True)
    seen = []

    def fn(logits, index):
        seen.append(logits)
        return torch.log_softmax(logits, -1).gather(-1, index.unsqueeze(-1)).squeeze(-1)

    loss, _ = call(kind, d, fn)
    loss.backward()
    # the reference's call order: new, ref, old
    want = [d['logit_new'], d['logit_ref'], d['logit_old']] if kind == 'grpo' else [d['logit_new'], d['logit_old']]
    assert all(a is b for a, b in zip(seen, want)) and len(seen) == len(want)
    assert dry.calls == ['b200rl_token_head_fwd', 'b200rl_scale']
    assert d['logit_new'].grad is not None


def test_lazy_info_returns_device_tensors(dry, monkeypatch):
    monkeypatch.setattr(R.ppo, 'LAZY_INFO', True)
    loss, info = call('grpo', go.make_case('grpo_f32_v2'))
    assert isinstance(info.approx_kl, torch.Tensor) and isinstance(info.clipfrac, torch.Tensor)
    assert not info.approx_kl.requires_grad


@pytest.mark.parametrize('dtype', [torch.float16, torch.float64])
def test_other_logit_dtypes_raise(dry, dtype):
    d = go.make_case('grpo_f32_v33')
    for k in ('logit_new', 'logit_old', 'logit_ref'):
        d[k] = d[k].to(dtype)
    with pytest.raises(TypeError, match='float32 or bfloat16'):
        call('grpo', d)
    with pytest.raises(TypeError, match='float32 or bfloat16'):
        R.naive_method(d['logit_new'], d['action'])


def test_mixed_logit_dtypes_raise(dry):
    d = go.make_case('rloo_f32_k2')
    d['logit_old'] = d['logit_old'].bfloat16()
    with pytest.raises(TypeError, match='share a dtype'):
        call('rloo', d)


@pytest.mark.parametrize('field,value', [
    ('action', torch.zeros(4, 7, dtype=torch.long)),
    ('weight', torch.ones(4, 9)),
    ('adv', torch.zeros(5)),
    ('logit_old', torch.zeros(4, 8, 999)),
])
def test_shape_errors(dry, field, value):
    d = go.make_case('grpo_f32_small')
    d[field] = value
    with pytest.raises(RuntimeError):
        call('grpo', d)


def test_rloo_reward_must_cover_the_batch(dry):
    d = go.make_case('rloo_f32_k2')
    d['reward'] = torch.zeros(3, 2)
    with pytest.raises(RuntimeError, match='reward'):
        call('rloo', d)


def test_log_prob_index_shape_error(dry):
    with pytest.raises(RuntimeError, match='index shape'):
        R.efficient_method(torch.zeros(2, 3, 5), torch.zeros(2, 4, dtype=torch.long))


@pytest.mark.parametrize('name', sorted(go.CASES))
def test_restatement_matches_the_reference_fixtures(name):
    """the float64 restatement on the fixture's inputs against the reference's outputs: 1e-5 on fp32 inputs; on bf16 the
    reference rounds each step to bf16, so the bar there is bf16's"""
    d = go.make_case(name)
    g = gold(name)
    np.testing.assert_allclose(g['checksum'], go.checksum(d), rtol=1e-12)
    want = go.run64(d)
    tol = 1e-5 if go.CASES[name][5] == torch.float32 else 2e-2
    for k in ('loss', 'approx_kl', 'clipfrac'):
        close(g[k], want[k], tol if k != 'clipfrac' else BF16_CLIPFRAC_TOL.get(go.CASES[name][5], tol))
    close(g['lp_new'], want['lp_new'].numpy(), tol)
    grad = go.grad_rows64(d['logit_new'], d['action'], want['dlp']).reshape(-1).numpy()
    if 'grad' in g:
        close(g['grad'], grad, tol)
    else:
        close(g['grad_sample'], grad[g['grad_index']], tol)


def test_restatement_matches_the_live_reference():
    with live_reference() as ref:
        for name in ('grpo_f32_mask', 'rloo_f32_k8_mask'):
            d = go.make_case(name)
            x = d['logit_new'].clone().requires_grad_(True)
            if 'logit_ref' in d:
                loss, info = ref['grpo'].grpo_policy_error(ref['grpo'].grpo_policy_data(
                    x, d['logit_old'], d['logit_ref'], d['action'], d['adv'], d['weight']))
            else:
                loss, info = ref['rloo'].rloo_policy_error(ref['rloo'].rloo_policy_data(
                    x, d['logit_old'], d['action'], d['reward'], d['weight']))
            loss.backward()
            want = go.run64(d)
            close(loss.item(), want['loss'], 1e-5)
            close(info.approx_kl, want['approx_kl'], 1e-5)
            close_grad(x.grad, go.grad_rows64(d['logit_new'], d['action'], want['dlp']), want['scale'], False)


def test_signatures_and_namedtuples_match_the_live_reference():
    with live_reference() as ref:
        for name in R.LM_HOT_PATH_FUNCTIONS:
            theirs = next(getattr(m, name) for m in ref.values() if hasattr(m, name))
            po, pt = inspect.signature(getattr(R, name)).parameters, inspect.signature(theirs).parameters
            assert list(po) == list(pt), name
            for k in po:
                a, b = po[k].default, pt[k].default
                assert (getattr(a, '__name__', a) == getattr(b, '__name__', b)), (name, k)
        for name in R.LM_HOT_PATH_TYPES:
            theirs = next(getattr(m, name) for m in ref.values() if hasattr(m, name))
            assert getattr(R, name)._fields == theirs._fields, name
        for name in ('naive_method', 'efficient_method', 'less_efficient_method'):
            assert R.log_prob_utils.is_fused(getattr(ref['log_prob_utils'], name))
            assert R.log_prob_utils.is_fused(getattr(R, name))
        assert not R.log_prob_utils.is_fused(lambda x, a: x)


def test_install_rebinds_the_language_model_losses(monkeypatch):
    monkeypatch.setattr(ops, 'require_cuda', lambda: None)
    with live_reference() as ref:
        for m in LM_MODULES:
            sys.modules['ding.rl_utils.' + m] = ref[m]
        originals = {(m, n): getattr(ref[m], n) for m in LM_MODULES for n in R.LM_HOT_PATH_FUNCTIONS
                     if hasattr(ref[m], n)}
        try:
            done = set(b2.install())
            for (m, n) in originals:
                assert ('ding.rl_utils.' + m, n) in done, (m, n)
                assert getattr(ref[m], n) is getattr(R, n)
        finally:
            b2.uninstall()
        for (m, n), fn in originals.items():
            assert getattr(ref[m], n) is fn


# ----------------------------------------------------------------------------------------------------------------
# GPU
# ----------------------------------------------------------------------------------------------------------------
DEV = 'cuda:0'


def to_dev(d):
    return {k: (v.to(DEV) if isinstance(v, torch.Tensor) else v) for k, v in d.items()}


def run_ours(kind, d, fn=None, g=None):
    d = dict(d)
    d['logit_new'] = d['logit_new'].clone().requires_grad_(True)
    loss, info = call(kind, d, fn)
    (loss if g is None else loss * g).backward()
    return loss.item(), info, d['logit_new'].grad


@pytest.mark.gpu
@pytest.mark.parametrize('name', sorted(go.CASES))
def test_kernel_against_fixtures_restatement_and_reference(name):
    kind, dtype = go.CASES[name][0], go.CASES[name][5]
    bf16 = dtype == torch.bfloat16
    d = to_dev(go.make_case(name))
    g = gold(name)
    loss, info, grad = run_ours(kind, d)
    lp = R.efficient_method(d['logit_new'], d['action'])
    want, grad64 = want64(d)
    # against the float64 restatement: 1e-5, the gradient entry by entry at its own size
    close(loss, want['loss'], 1e-5)
    close(info.approx_kl, want['approx_kl'], 1e-5)
    close(info.clipfrac, want['clipfrac'], 1e-5)
    close(lp.cpu().numpy(), want['lp_new'].cpu().numpy(), 1e-5)
    close_grad(grad, grad64, want['scale'], bf16)
    # against the reference's outputs: the fixture (reference on the CPU) and, where it is importable, the reference run
    # on the same CUDA tensors.  fp32: the same bars; bf16: the reference rounds every step to bf16
    tol = 2e-2 if bf16 else 1e-5
    outs = [(g['loss'], g['approx_kl'], g['clipfrac'], g['lp_new'], g.get('grad'), g.get('grad_index'),
             g.get('grad_sample'))]
    from oracle import ref_lm
    if ref_lm.available():
        with ref_lm.modules() as ref:
            r_loss, r_info, r_grad = ref_call(ref, kind, d)
            r_lp = ref['log_prob_utils'].efficient_method(d['logit_new'], d['action']).float().cpu().numpy()
        outs.append((r_loss, r_info.approx_kl, r_info.clipfrac, r_lp, r_grad, None, None))
    for r_loss, r_kl, r_cf, r_lp, r_grad, r_idx, r_sample in outs:
        close(loss, r_loss, tol)
        close(info.approx_kl, r_kl, tol)
        close(info.clipfrac, r_cf, BF16_CLIPFRAC_TOL.get(dtype, tol))
        close(lp.cpu().numpy(), r_lp, tol)
        if r_grad is not None:
            r_grad = torch.as_tensor(np.asarray(r_grad.float().cpu() if torch.is_tensor(r_grad) else r_grad))
            if bf16:
                close(grad.float().cpu().numpy().reshape(-1), r_grad.numpy().reshape(-1), tol)
            else:
                close_grad(grad, r_grad.to(DEV).reshape(grad.shape), want['scale'], False)
        else:
            close(grad.float().reshape(-1).cpu().numpy()[r_idx], r_sample, tol)


@pytest.mark.gpu
@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
@pytest.mark.parametrize('shape', [(2, 3, 2), (4, 9, 1027), (3, 5, 32771), (7, 129)])
@pytest.mark.parametrize('method', ['naive_method', 'efficient_method', 'less_efficient_method'])
def test_log_prob_methods(dtype, shape, method):
    gen = torch.Generator().manual_seed(sum(shape))
    x = (torch.randn(*shape, generator=gen) * 3).to(dtype).to(DEV).requires_grad_(True)
    idx = torch.randint(0, shape[-1], shape[:-1], generator=gen).to(DEV)
    lp = getattr(R, method)(x, idx)
    want = go.logp64(x.detach(), idx)
    close(lp.detach().cpu().numpy(), want.cpu().numpy(), 1e-5)
    up = torch.randn(shape[:-1], generator=gen).to(DEV)
    (lp * up).sum().backward()
    g64 = go.grad_rows64(x.detach(), idx, up.double())
    close_grad(x.grad, g64, up, dtype == torch.bfloat16)


@pytest.mark.gpu
@pytest.mark.parametrize('name', ['grpo_f32_mask', 'rloo_f32_k8_mask', 'grpo_bf16_mask'])
def test_scaled_and_repeated_backward(name):
    kind = go.CASES[name][0]
    bf16 = go.CASES[name][5] == torch.bfloat16
    d = to_dev(go.make_case(name))
    want, grad64 = want64(d)
    _, _, g1 = run_ours(kind, d)
    _, _, g25 = run_ours(kind, d, g=2.5)
    close_grad(g1, grad64, want['scale'], bf16)
    close_grad(g25, 2.5 * grad64, 2.5 * want['scale'], bf16)
    x = d['logit_new'].clone().requires_grad_(True)
    loss, _ = call(kind, dict(d, logit_new=x))
    loss.backward(retain_graph=True)
    first = x.grad.clone()
    loss.backward()
    close_grad(x.grad, 2 * grad64, 2 * want['scale'], bf16)
    assert torch.equal(first, g1)  # the forward-written gradient, bit for bit


@pytest.mark.gpu
@pytest.mark.parametrize('name', ['grpo_f32_mask', 'rloo_f32_k2_zero_row', 'grpo_bf16_small'])
def test_custom_log_prob_fn(name):
    kind = go.CASES[name][0]
    d = to_dev(go.make_case(name))

    def fn(logits, index):
        return torch.log_softmax(logits.float(), -1).gather(-1, index.unsqueeze(-1)).squeeze(-1)

    want, grad64 = want64(d)
    loss_f, info_f, grad_f = run_ours(kind, d)
    loss_c, info_c, grad_c = run_ours(kind, d, fn)
    close(loss_c, loss_f, 1e-5)
    close(info_c.approx_kl, info_f.approx_kl, 1e-5)
    close(info_c.clipfrac, info_f.clipfrac, 0.0)
    close_grad(grad_c, grad64, want['scale'], go.CASES[name][5] == torch.bfloat16)


def _edge_lp():
    """d with fp32 exp(d) = fp32(1 + clip) and e with exp(e) = fp32(1 - clip), each within a tenth of an ulp in float64,
    so that every faithful expf lands on the bound itself"""
    out = []
    for bound in (np.float32(1 + go.CLIP), np.float32(1 - go.CLIP)):
        d0 = np.float32(np.log(np.float64(bound)))
        cands = [np.float32(d0) + np.float32(k) * np.spacing(d0) for k in range(-8, 9)]
        best = min(cands, key=lambda c: abs(np.exp(np.float64(c)) - np.float64(bound)))
        assert abs(np.exp(np.float64(best)) - np.float64(bound)) < 0.1 * np.spacing(bound)
        out.append(float(best))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize('kind', ['grpo', 'rloo'])
def test_ratio_exactly_at_the_clip_bounds(kind):
    """through the token head (a custom log_prob_fn that returns its input): ratios at fp32(1 -+ clip) and 1 with
    positive, negative and zero advantages -- min() ties, clamp() edges, the clipfrac comparisons -- against the
    reference's own arithmetic in fp32"""
    hi, lo = _edge_lp()
    B, S = 4, 6
    lp_new = torch.tensor([[hi, lo, 0.0, hi, lo, 0.3]] * B, dtype=torch.float32)
    lp_old = torch.zeros(B, S)
    lp_ref = torch.full((B, S), -0.25)
    action = torch.zeros(B, S, dtype=torch.long)
    weight = torch.tensor([[1., 1., 0., 1., 1., 1.]] * B)
    ident = lambda x, a: x  # noqa: E731
    if kind == 'grpo':
        adv = torch.tensor([1.0, -1.0, 0.0, 2.0])
        adv_eff, ref_lp = adv, lp_ref
    else:
        reward = torch.tensor([[1.0, -2.0], [0.5, 0.5]])
        adv_eff, ref_lp = go.rloo_adv64(reward).float(), None
    x = lp_new.clone().requires_grad_(True)
    want_loss, want_kl, want_cf = go.head64(x, lp_old, ref_lp, adv_eff, weight, go.CLIP, go.BETA if ref_lp is not None else 0.0)
    want_loss.backward()
    xd = lp_new.to(DEV).requires_grad_(True)
    if kind == 'grpo':
        data = R.grpo_policy_data(xd, lp_old.to(DEV), lp_ref.to(DEV), action.to(DEV), adv.to(DEV), weight.to(DEV))
        loss, info = R.grpo_policy_error(data, ident)
    else:
        data = R.rloo_policy_data(xd, lp_old.to(DEV), action.to(DEV), reward.to(DEV), weight.to(DEV))
        loss, info = R.rloo_policy_error(data, ident)
    loss.backward()
    close(loss.item(), want_loss.item(), 1e-6)
    close(info.approx_kl, want_kl.item(), 1e-6)
    assert info.clipfrac == pytest.approx(want_cf.item(), abs=0)
    close(xd.grad.cpu().numpy(), x.grad.numpy(), 1e-6)


@pytest.mark.gpu
@pytest.mark.parametrize('shape,dtype', [((16, 1024, 32768), torch.float32), ((16, 1024, 32768), torch.bfloat16),
                                         ((4, 128, 152064), torch.bfloat16)])
@pytest.mark.parametrize('kind', ['grpo', 'rloo'])
def test_language_model_scale(shape, dtype, kind):
    B, S, V = shape
    gen = torch.Generator(device=DEV).manual_seed(B + S + V)
    new = torch.randn(B, S, V, device=DEV, generator=gen, dtype=dtype) * 2
    d = {'logit_new': new, 'logit_old': (new.float() + 0.1 * torch.randn(B, S, V, device=DEV, generator=gen)).to(dtype),
         'action': torch.randint(0, V, (B, S), device=DEV, generator=gen),
         'weight': (torch.rand(B, S, device=DEV, generator=gen) > 0.2).float()}
    if kind == 'grpo':
        d['logit_ref'] = (new.float() + 0.2 * torch.randn(B, S, V, device=DEV, generator=gen)).to(dtype)
        d['adv'] = torch.randn(B, device=DEV, generator=gen)
    else:
        d['reward'] = torch.randn(2, B // 2, device=DEV, generator=gen)
    bf16 = dtype == torch.bfloat16
    loss, info, grad = run_ours(kind, d)
    want = go.run64(d)
    close(loss, want['loss'], 1e-5)
    close(info.approx_kl, want['approx_kl'], 1e-5)
    close(info.clipfrac, want['clipfrac'], 1e-5)
    for b in range(B):  # every row, each entry at its own size
        g64 = go.grad_rows64(d['logit_new'][b], d['action'][b], want['dlp'][b])
        close_grad(grad[b], g64, want['scale'][b], bf16)
    del g64
    # the reference itself, with its default efficient_method, on the same CUDA tensors
    from oracle import ref_lm
    if not ref_lm.available():
        return
    with ref_lm.modules() as ref:
        r_loss, r_info, r_grad = ref_call(ref, kind, d)
    tol = 2e-2 if bf16 else 1e-5
    close(loss, r_loss, tol)
    close(info.approx_kl, r_info.approx_kl, tol)
    close(info.clipfrac, r_info.clipfrac, BF16_CLIPFRAC_TOL.get(dtype, tol))
    if not bf16:
        close_grad(grad, r_grad, want['scale'], False)


@pytest.mark.gpu
def test_host_tensors():
    d = go.make_case('grpo_f32_mask')
    loss_h, info_h, grad_h = run_ours('grpo', d)
    loss_d, info_d, grad_d = run_ours('grpo', to_dev(d))
    assert grad_h.device.type == 'cpu'
    close(loss_h, loss_d, 0.0)
    close(grad_h.numpy(), grad_d.cpu().numpy(), 0.0)


# the reference's own tests (ding/rl_utils/tests/test_grpo_rlhf.py, test_rloo_rlhf.py, test_log_prob_utils.py), run
# against this library's functions on the GPU
@pytest.mark.gpu
@pytest.mark.parametrize('masked', [False, True])
def test_ported_grpo_policy_loss(masked, batch_size=4, seq_length=8, vocab_size=1000):
    logit_new = torch.randn(batch_size, seq_length, vocab_size, device=DEV).requires_grad_(True)
    logit_old = logit_new + torch.randn_like(logit_new) * 0.1
    logit_ref = logit_new + torch.randn_like(logit_new) * 0.2
    action = torch.randint(0, vocab_size, (batch_size, seq_length), device=DEV)
    adv = torch.randn(batch_size, device=DEV)
    weight = None
    if masked:
        weight = torch.ones(batch_size, seq_length, device=DEV)
        weight[:, -2:] = 0
    data = R.grpo_policy_data(logit_new=logit_new, logit_old=logit_old, logit_ref=logit_ref, action=action, adv=adv,
                              weight=weight)
    loss, info = R.grpo_policy_error(data=data, clip_ratio=0.2, beta=0.1)
    assert isinstance(loss, torch.Tensor) and loss.shape == torch.Size([])
    assert not torch.isnan(loss) and not torch.isinf(loss)
    assert logit_new.grad is None
    loss.backward()
    assert isinstance(logit_new.grad, torch.Tensor)
    assert 'approx_kl' in info._asdict() and 'clipfrac' in info._asdict()
    assert all([np.isscalar(v) for v in info._asdict().values()])


@pytest.mark.gpu
@pytest.mark.parametrize('masked', [False, True])
def test_ported_rloo_policy_loss(masked, batch_size=4, seq_length=8, dictionary_num=1000):
    logit_new = torch.randn(batch_size, seq_length, dictionary_num, device=DEV).requires_grad_(True)
    logit_old = logit_new + torch.randn_like(logit_new) * 0.1
    action = torch.randint(0, dictionary_num, (batch_size, seq_length), device=DEV)
    reward = torch.randn(batch_size, device=DEV)
    action_mask = torch.ones(batch_size, seq_length, device=DEV) if masked else None
    if masked:
        action_mask[:, -2:] = 0
    data = R.rloo_policy_data(logit_new=logit_new, logit_old=logit_old, action=action, reward=reward,
                              weight=action_mask)
    loss, info = R.rloo_policy_error(data, clip_ratio=0.2)
    assert isinstance(loss, torch.Tensor) and loss.shape == torch.Size([])
    assert not torch.isnan(loss) and not torch.isinf(loss)
    assert logit_new.grad is None
    loss.backward()
    assert isinstance(logit_new.grad, torch.Tensor)
    assert 'approx_kl' in info._asdict() and 'clipfrac' in info._asdict()
    assert all([np.isscalar(v) for v in info._asdict().values()])


@pytest.mark.gpu
@pytest.mark.parametrize('dtype,tolerance', [(torch.float32, 1e-5), (torch.bfloat16, 1e-1)])
def test_ported_log_prob_methods(dtype, tolerance, batch_size=16, seq_length=1024, dictionary_num=32768):
    logits = torch.randn(batch_size, seq_length, dictionary_num, device=DEV, dtype=dtype)
    input_ids = torch.randint(0, dictionary_num, (batch_size, seq_length), device=DEV)
    results = {name: getattr(R, name)(logits, input_ids) for name in ('naive_method', 'efficient_method',
                                                                      'less_efficient_method')}
    ref = results['naive_method']
    for name, r in results.items():
        assert r.shape == ref.shape
        diff = (r - ref).abs().max().item()
        assert diff < tolerance, name
    expect = torch.log_softmax(logits.float(), -1).gather(-1, input_ids.unsqueeze(-1)).squeeze(-1)
    assert (ref - expect).abs().max().item() < 1e-4
