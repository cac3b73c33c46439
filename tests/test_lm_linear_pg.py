"""ppo_policy_error_linear and a2c_error_linear (rl_utils/lm_linear.py): PPO and A2C from the lm_head's hidden states, the
logits one chunk of token rows at a time, the loss mix one differentiable output.

CPU, on the recording stand-in of tests/test_lm_linear.py: argument, dtype and mix-weight errors, the chunk plan with
PPO's five partial sums (and a plan that raises before any launch), a row range that crosses chunk boundaries, gradient
GEMMs only for the inputs that require grad, A2C's value gradient alone, and that no (B*S, V) tensor is ever allocated.

GPU: the loss, every component, approx_kl, clipfrac, d hidden, d lm_weight and (A2C) d value against the library's own
composition (F.linear + ppo_policy_error / a2c_error on the logits) and against a float64 restatement
(tests/ppo_lm_oracle.run64, oracle/rl_oracle.a2c_error; d / d logits mapped through W and H in float64), with the rules of
tests/test_lm_linear.py: fp32 1e-5, bf16 2 * the composition's error.  Also: an all-zero mask row, one input requiring
grad, a tied weight, an upstream gradient != 1 with a second backward, bit-identical repeats, a compiled learner step and
peak memory."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import di_engine_b200 as b2
from di_engine_b200 import ops
from oracle import rl_oracle
from tests import ppo_lm_oracle as po
from tests.test_lm_linear import _Ops, check_scalar, check_tensor, dry  # noqa: F401  (dry: the recording fixture)

R = b2.rl_utils
B_, S_, D_, V_ = 3, 100, 8, 1031  # 300 rows: chunks of 128, 128 and 44 rows when the budget holds 128 rows
EW, KW, VW = 0.01, 0.1, 0.5  # entropy_weight, kl_weight, value_weight


def make(dtype=torch.float32, B=B_, S=S_, D=D_, V=V_, weight=True, pre=True, seed=0):
    g = torch.Generator().manual_seed(seed)
    return {
        'hidden': torch.randn(B, S, D, generator=g).to(dtype),
        'lm_weight': (torch.randn(V, D, generator=g) / D ** 0.5).to(dtype),
        'action': torch.randint(0, V, (B, S), generator=g),
        'logp_old': -torch.rand(B, S, generator=g) * 6 - 1,
        'logp_pretrained': -torch.rand(B, S, generator=g) * 6 - 1 if pre else None,
        'adv': torch.randn(B, S, generator=g),
        'value': torch.randn(B, S, generator=g),
        'return_': torch.randn(B, S, generator=g),
        'weight': (torch.rand(B, S, generator=g) > 0.2).float() if weight else None,
    }


def ppo_call(d, **kw):
    return R.ppo_policy_error_linear(R.ppo_policy_linear_data(d['hidden'], d['lm_weight'], d['logp_old'], d['action'],
                                                              d['adv'], d['weight'], d['logp_pretrained']), **kw)


def a2c_call(d, **kw):
    return R.a2c_error_linear(R.a2c_linear_data(d['hidden'], d['lm_weight'], d['action'], d['value'], d['adv'],
                                                d['return_'], d['weight']), **kw)


@pytest.fixture
def rows128(monkeypatch):
    monkeypatch.setattr(ops, 'LM_CHUNK_BYTES', 128 * V_ * 4)


# ----------------------------------------------------------------------------------------------------------------
# CPU
# ----------------------------------------------------------------------------------------------------------------
# b200rl_lm_linear_pg_fwd's arguments by position
A_MODE, A_ROW0, A_ROWS, A_CHUNK, A_N, A_LPO, A_LPP, A_VAL, A_RET = 0, 3, 4, 5, 7, 9, 10, 12, 13
A_KL, A_ENT, A_WENT, A_WKL, A_WVAL, A_DV, A_WANT = 17, 18, 19, 20, 21, 22, 24


@pytest.mark.filterwarnings('ignore:invalid value encountered in cast')  # the stand-in leaves outputs uninitialised
@pytest.mark.parametrize('kind', ['ppo', 'ppo_noent_nopre', 'a2c'])
@pytest.mark.parametrize('grads', [(True, True), (True, False), (False, True), (False, False)])
def test_loss_wiring_and_chunks(dry, rows128, kind, grads):
    """one row launch per chunk at rows [0, 128), [128, 256), [256, 300) with the loss mix as launch arguments; a dH GEMM
    per chunk only if hidden requires grad, a dW GEMM only if lm_weight does; an in-place scale of each at backward; no
    sequence-normaliser launch; and never a (B*S, V) tensor"""
    d = make(pre=kind != 'ppo_noent_nopre')
    d['hidden'].requires_grad_(grads[0])
    d['lm_weight'].requires_grad_(grads[1])
    with _Ops() as rec:
        if kind == 'a2c':
            loss = a2c_call(d, value_weight=VW, entropy_weight=EW)
        elif kind == 'ppo':
            loss, info = ppo_call(d, dual_clip=2.0, kl_type='k3', entropy_weight=EW, kl_weight=KW)
        else:
            loss, info = ppo_call(d, entropy_bonus=False)
        if any(grads):
            loss.loss.backward()
    fwd = [c[1] for c in dry.calls if c[0] == 'b200rl_lm_linear_pg_fwd']
    assert dry.names() == ['b200rl_lm_linear_pg_fwd'] * 3 + ['b200rl_lm_linear_scale'] * sum(grads)
    assert [(c[A_ROW0], c[A_ROWS], c[A_CHUNK], c[A_N]) for c in fwd] == [(0, 128, 128, 300), (128, 128, 128, 300),
                                                                         (256, 44, 128, 300)]
    mode = {'ppo': 3, 'ppo_noent_nopre': 3, 'a2c': 4}[kind]
    mix = {'ppo': (1, -EW, KW, 0.0), 'ppo_noent_nopre': (0, 0.0, 0.0, 0.0), 'a2c': (1, -EW, 0.0, VW)}[kind]
    for c in fwd:
        assert c[A_MODE] == mode and c[A_WANT] == int(any(grads))
        assert (c[A_ENT], c[A_WENT], c[A_WKL], c[A_WVAL]) == mix
        assert c[A_DV] is None  # value does not require grad here
        assert (c[A_LPP] is None) == (kind != 'ppo') and (c[A_LPO] is None) == (kind == 'a2c')
        assert (c[A_VAL] is None) == (kind != 'a2c') and (c[A_RET] is None) == (kind != 'a2c')
    if kind == 'ppo':
        assert all(c[A_KL] == 3 for c in fwd)
    assert rec.count('mm') == 3 + 3 * grads[0]
    assert rec.count('addmm', 'addmm_') == 3 * grads[1]
    assert all(int(np.prod(s)) < B_ * S_ * V_ for s in rec.allocated())
    assert sum(1 for s in rec.allocated() if s == (128, V_)) == 1  # one chunk buffer per call
    assert loss.loss.requires_grad == any(grads)
    for x in loss[1:]:
        assert x.dim() == 0 and not x.requires_grad
    if kind != 'a2c':
        assert isinstance(info.approx_kl, float) and isinstance(info.clipfrac, float)
    if grads[0]:
        assert d['hidden'].grad.shape == d['hidden'].shape
    if grads[1]:
        assert d['lm_weight'].grad.shape == (V_, D_)
    if not any(grads):
        assert (B_ * S_, D_) not in rec.allocated() and (V_, D_) not in rec.allocated()


@pytest.mark.filterwarnings('ignore:invalid value encountered in cast')
@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
def test_a2c_value_gradient_alone(dry, rows128, dtype):
    """only value requires grad: the launches compute d value (no in-place logit gradient), no dH / dW GEMM, one scale
    (of d value, fp32); a bf16 value gets its gradient back in bf16"""
    d = make()
    d['value'] = d['value'].to(dtype).requires_grad_(True)
    with _Ops() as rec:
        loss = a2c_call(d)
        loss.loss.backward()
    fwd = [c[1] for c in dry.calls if c[0] == 'b200rl_lm_linear_pg_fwd']
    assert len(fwd) == 3 and all(c[A_WANT] == 0 and c[A_DV] is not None for c in fwd)
    assert len({c[A_DV] for c in fwd}) == 1  # one (B*S) buffer, written at the global rows
    scales = [c[1] for c in dry.calls if c[0] == 'b200rl_lm_linear_scale']
    assert len(scales) == 1 and scales[0][0] == 0 and scales[0][3] == B_ * S_
    assert rec.count('mm') == 3 and rec.count('addmm', 'addmm_') == 0
    assert d['value'].grad.shape == (B_, S_) and d['value'].grad.dtype == dtype


@pytest.mark.filterwarnings('ignore:invalid value encountered in cast')
def test_a2c_all_three_gradients(dry, rows128):
    d = make()
    for k in ('hidden', 'lm_weight', 'value'):
        d[k].requires_grad_(True)
    a2c_call(d).loss.backward()
    fwd = [c[1] for c in dry.calls if c[0] == 'b200rl_lm_linear_pg_fwd']
    assert all(c[A_WANT] == 1 and c[A_DV] is not None for c in fwd)
    assert dry.names().count('b200rl_lm_linear_scale') == 3
    assert d['value'].grad.shape == (B_, S_)


@pytest.mark.filterwarnings('ignore:invalid value encountered in cast')
def test_no_grad_allocates_no_gradient_buffer(dry, rows128):
    d = make()
    for k in ('hidden', 'lm_weight', 'value'):
        d[k].requires_grad_(True)
    with torch.no_grad(), _Ops() as rec:
        loss = a2c_call(d)
        ppo_call(d)
    assert not loss.loss.requires_grad
    assert all(c[1][A_WANT] == 0 and c[1][A_DV] is None for c in dry.calls)
    assert (B_ * S_, D_) not in rec.allocated() and (V_, D_) not in rec.allocated() and (B_ * S_, ) not in rec.allocated()


def test_chunk_plan_with_five_partials(monkeypatch):
    monkeypatch.setattr(ops, 'LM_CHUNK_BYTES', 1)
    # 128-row chunks: 128 CTAs x 5 partials each; 399 chunks fit below the workspace's 255 984 partial words, 400 do not
    assert ops.lm_chunk_plan(399 * 128, 50, 4, 132, True, 5) == (128, 399)
    with pytest.raises(ValueError, match='partials'):
        ops.lm_chunk_plan(400 * 128, 50, 4, 132, True, 5)
    assert ops.lm_chunk_plan(400 * 128, 50, 4, 132, True) == (128, 400)  # 3 sums (GRPO, RLOO, A2C) still fit
    assert ops.lm_chunk_plan(400 * 128, 50, 4, 132, True, 3) == (128, 400)


def test_partials_overflow_raises_before_any_launch(dry, monkeypatch):
    """400 chunks of 128 rows: PPO's five partials do not fit, A2C's three do"""
    monkeypatch.setattr(ops, 'LM_CHUNK_BYTES', 1)
    d = make(B=2, S=400 * 64, D=2, V=3, weight=False)
    with pytest.raises(ValueError, match='partials'):
        ppo_call(d)
    assert dry.calls == []
    a2c_call(d)
    assert dry.names() == ['b200rl_lm_linear_pg_fwd'] * 400


@pytest.mark.parametrize('dtype', [torch.float16, torch.float64])
def test_other_dtypes_raise(dry, dtype):
    d = make()
    d['hidden'], d['lm_weight'] = d['hidden'].to(dtype), d['lm_weight'].to(dtype)
    with pytest.raises(TypeError, match='float32 or both bfloat16'):
        ppo_call(d)
    with pytest.raises(TypeError, match='float32 or both bfloat16'):
        a2c_call(d)
    assert dry.calls == []


def test_mixed_dtypes_raise(dry):
    d = make()
    d['lm_weight'] = d['lm_weight'].bfloat16()
    for call in (ppo_call, a2c_call):
        with pytest.raises(TypeError, match='both'):
            call(d)


@pytest.mark.filterwarnings('ignore:invalid value encountered in cast')
def test_side_inputs_of_any_float_dtype_are_read_as_fp32(dry):
    d = make()
    for k in ('logp_old', 'logp_pretrained', 'weight', 'return_'):
        d[k] = d[k].double()
    d['adv'] = d['adv'].bfloat16()
    d['value'] = d['value'].half()
    ppo_call(d)
    a2c_call(d)
    assert dry.names() == ['b200rl_lm_linear_pg_fwd'] * 2


@pytest.mark.parametrize('field,value,err', [
    ('hidden', torch.zeros(300, 8), 'hidden must be'),
    ('lm_weight', torch.zeros(1031, 9), 'lm_weight must be'),
    ('lm_weight', torch.zeros(1031), 'lm_weight must be'),
    ('action', torch.zeros(3, 99, dtype=torch.long), 'action must be'),
    ('weight', torch.ones(3, 101), 'weight must be'),
    ('adv', torch.zeros(3), 'adv must be'),
    ('logp_old', torch.zeros(3, 99), 'logp_old must be'),
    ('logp_pretrained', torch.zeros(300), 'logp_pretrained must be'),
    ('value', torch.zeros(3, 99), 'value must be'),
    ('return_', torch.zeros(300), 'return_ must be'),
])
def test_argument_errors(dry, field, value, err):
    d = make()
    d[field] = value
    call = a2c_call if field in ('value', 'return_') else ppo_call
    with pytest.raises(RuntimeError, match=err):
        call(d)
    assert dry.calls == []


def test_option_and_mix_weight_errors(dry):
    d = make()
    with pytest.raises(AssertionError, match='dual_clip'):
        ppo_call(d, dual_clip=1.0)
    with pytest.raises(ValueError, match='Unknown kl_type'):
        ppo_call(d, kl_type='k4')
    with pytest.raises(ValueError, match='entropy_bonus'):
        ppo_call(d, entropy_bonus=False, entropy_weight=0.01)
    with pytest.raises(ValueError, match='logp_pretrained'):
        ppo_call(dict(d, logp_pretrained=None), kl_weight=0.1)
    assert dry.calls == []


@pytest.mark.filterwarnings('ignore:invalid value encountered in cast')
def test_unknown_kl_type_without_pretrained_is_unused(dry):
    """as ppo_policy_error: kl_type is only looked at with a pretrained policy"""
    ppo_call(dict(make(), logp_pretrained=None), kl_type='k4')
    assert dry.names() == ['b200rl_lm_linear_pg_fwd']


def test_out_of_range_action_raises_with_index_checks(dry, monkeypatch):
    monkeypatch.setattr(ops, 'CHECK_INDICES', True)
    d = make()
    d['action'][1, 7] = V_
    for call in (ppo_call, a2c_call):
        with pytest.raises(IndexError, match='out of range'):
            call(d)
    assert dry.calls == []


@pytest.mark.filterwarnings('ignore:invalid value encountered in cast')
def test_lazy_info(dry, monkeypatch):
    monkeypatch.setattr(R.ppo, 'LAZY_INFO', True)
    _, info = ppo_call(make())
    assert isinstance(info.approx_kl, torch.Tensor) and info.approx_kl.dim() == 0


def test_exports_stay_outside_the_reference_lists():
    for name in ('ppo_policy_error_linear', 'a2c_error_linear', 'ppo_policy_linear_data', 'ppo_linear_loss',
                 'a2c_linear_data', 'a2c_linear_loss'):
        assert getattr(R, name) is not None
        assert name not in R.HOT_PATH_FUNCTIONS and name not in R.LM_HOT_PATH_FUNCTIONS
        assert name not in R.COMA_HOT_PATH_FUNCTIONS


# ----------------------------------------------------------------------------------------------------------------
# GPU
# ----------------------------------------------------------------------------------------------------------------
gpu = pytest.mark.gpu
PPO_OPTS = {  # name -> dual_clip, kl_type (None: no logp_pretrained), entropy_bonus, mask
    'k3_ent': (None, 'k3', True, True),
    'dc_k1_ent': (2.0, 'k1', True, True),
    'k2_noent': (None, 'k2', False, True),
    'nopre_ent_noweight': (None, None, True, False),
}


def gpu_case(dtype, B, S, D, V, seed=0, mask=True, pre=True, zero_row=False):
    """hidden / lm_weight on the device, and logp_old / logp_pretrained from perturbed hidden states of the same head (so
    the ratios sit around 1 and some clip); the logit tensors of the composition are kept for it"""
    torch.manual_seed(seed)
    dev = torch.device('cuda')
    h = (torch.randn(B, S, D, device=dev) * 2).to(dtype)
    w = torch.randn(V, D, device=dev).div(D ** 0.5).to(dtype)
    action = torch.randint(0, V, (B, S), device=dev)
    h_old = (h.float() + 0.05 * torch.randn_like(h.float())).to(dtype)
    h_pre = (h.float() + 0.1 * torch.randn_like(h.float())).to(dtype)
    with torch.no_grad():
        logit_old, logit_pre = F.linear(h_old, w), F.linear(h_pre, w) if pre else None
        lp_old = R.efficient_method(logit_old, action)
        lp_pre = R.efficient_method(logit_pre, action) if pre else None
    weight = (torch.rand(B, S, device=dev) > 0.25).float() if mask else None
    if zero_row:
        weight[1] = 0
    adv = torch.randn(B, S, device=dev)
    adv[0, 0] = 0.0  # a tie of the min
    return {'hidden': h, 'lm_weight': w, 'action': action, 'logp_old': lp_old, 'logp_pretrained': lp_pre,
            'logit_old': logit_old, 'logit_pretrained': logit_pre, 'weight': weight, 'adv': adv,
            'value': torch.randn(B, S, device=dev), 'return_': torch.randn(B, S, device=dev)}


def _leaves(d, needs):
    h = d['hidden'].detach().clone().requires_grad_(needs[0])
    w = d['lm_weight'].detach().clone().requires_grad_(needs[1])
    v = d['value'].detach().clone().requires_grad_(needs[2] if len(needs) > 2 else False)
    return h, w, v


def ours(kind, d, opts, needs=(True, True, True)):
    """-> (scalars, d hidden, d lm_weight, d value)"""
    h, w, v = _leaves(d, needs)
    e = dict(d, hidden=h, lm_weight=w, value=v)
    if kind == 'ppo':
        dual, kl, ent = opts
        loss, info = ppo_call(e, dual_clip=dual, kl_type=kl or 'k1', entropy_bonus=ent, entropy_weight=EW if ent else 0.0,
                              kl_weight=KW if kl else 0.0)
        vals = [loss.loss.item(), loss.policy_loss.item(), loss.entropy_loss.item(), loss.kl_div.item(), info.approx_kl,
                info.clipfrac]
    else:
        loss = a2c_call(e, value_weight=VW, entropy_weight=EW)
        vals = [loss.loss.item(), loss.policy_loss.item(), loss.value_loss.item(), loss.entropy_loss.item()]
    loss.loss.backward()
    return vals, h.grad, w.grad, v.grad


def composition(kind, d, opts, needs=(True, True, True)):
    """F.linear + the library's logit losses, the same mix"""
    h, w, v = _leaves(d, needs)
    logits = F.linear(h, w)
    if kind == 'ppo':
        dual, kl, ent = opts
        p, info = R.ppo_policy_error(R.ppo_policy_data(logits, d['logit_old'], d['action'], d['adv'], d['weight'],
                                                       d['logit_pretrained']), po.CLIP, dual, ent, kl or 'k1')
        loss = p.policy_loss - (EW if ent else 0.0) * p.entropy_loss + (KW if kl else 0.0) * p.kl_div
        vals = [loss.item(), p.policy_loss.item(), float(p.entropy_loss), p.kl_div.item(), info.approx_kl, info.clipfrac]
    else:
        a = R.a2c_error(R.a2c_data(logits, d['action'], v, d['adv'], d['return_'], d['weight']))
        loss = a.policy_loss + VW * a.value_loss - EW * a.entropy_loss
        vals = [loss.item(), a.policy_loss.item(), a.value_loss.item(), a.entropy_loss.item()]
    loss.backward()
    return vals, h.grad, w.grad, v.grad


def fp64(kind, d, opts):
    """the float64 restatement: d / d logits mapped through W and H in float64"""
    h, w = d['hidden'].double(), d['lm_weight'].double()
    logits = h @ w.t()
    if kind == 'ppo':
        dual, kl, ent = opts
        c = {'logit_new': logits, 'logit_old': d['logit_old'], 'logit_pretrained': d['logit_pretrained'],
             'action': d['action'], 'adv': d['adv'], 'weight': d['weight']}
        mix = (1.0, -EW if ent else 0.0, KW if kl else 0.0)
        r = po.run64(c, po.CLIP, dual, kl or 'k1', ent, mix)
        vals = [mix[0] * r['policy'] + mix[1] * r['entropy'] + mix[2] * r['kl'], r['policy'], r['entropy'], r['kl'],
                r['approx_kl'], r['clipfrac']]
        g, gv = r['grad'], None
    else:
        x = logits.detach().requires_grad_(True)
        v = d['value'].double().requires_grad_(True)
        wt = d['weight'].double() if d['weight'] is not None else None
        p, vl, e = rl_oracle.a2c_error(x, d['action'], v, d['adv'].double(), d['return_'].double(), wt)
        loss = p + VW * vl - EW * e
        loss.backward()
        vals = [loss.item(), p.item(), vl.item(), e.item()]
        g, gv = x.grad, v.grad
    g = g.reshape(-1, g.shape[-1])
    return vals, (g @ w).reshape(h.shape), g.t() @ h.reshape(-1, h.shape[-1]), gv


def compare(kind, d, opts, needs=(True, True, True)):
    bf16 = d['hidden'].dtype == torch.bfloat16
    got, comp, want = ours(kind, d, opts, needs), composition(kind, d, opts, needs), fp64(kind, d, opts)
    N = d['action'].numel()
    for k in range(len(got[0])):
        check_scalar(got[0][k], comp[0][k], want[0][k], bf16, 2.0 / N if (kind == 'ppo' and k == 5) else 0.0)
    for k, need in zip((1, 2, 3), needs):
        if kind == 'ppo' and k == 3:
            continue
        if need:
            check_tensor(got[k], comp[k], want[k], bf16)
        else:
            assert got[k] is None
    return got


SIZES = [(torch.float32, 1003), (torch.bfloat16, 1003), (torch.float32, 32771), (torch.bfloat16, 32771),
         (torch.bfloat16, 152064)]


def _split(monkeypatch, split, V, dtype):
    if split:
        monkeypatch.setattr(ops, 'LM_CHUNK_BYTES', 128 * V * torch.tensor([], dtype=dtype).element_size())


@gpu
@pytest.mark.parametrize('opts', list(PPO_OPTS))
@pytest.mark.parametrize('dtype,V', SIZES)
@pytest.mark.parametrize('split', [False, True])
def test_ppo_against_composition_and_fp64(monkeypatch, opts, dtype, V, split):
    """split: 128-row chunks over 4 x 75 tokens (300 is no multiple of the chunk)"""
    _split(monkeypatch, split, V, dtype)
    dual, kl, ent, mask = PPO_OPTS[opts]
    compare('ppo', gpu_case(dtype, 4, 75, 64, V, mask=mask, pre=kl is not None), (dual, kl, ent))


@gpu
@pytest.mark.parametrize('weight', [True, False])
@pytest.mark.parametrize('dtype,V', SIZES)
@pytest.mark.parametrize('split', [False, True])
def test_a2c_against_composition_and_fp64(monkeypatch, weight, dtype, V, split):
    _split(monkeypatch, split, V, dtype)
    compare('a2c', gpu_case(dtype, 4, 75, 64, V, mask=weight, pre=False), None)


@gpu
@pytest.mark.parametrize('kind', ['ppo', 'a2c'])
def test_all_zero_mask_row(monkeypatch, kind):
    """a sequence whose mask is all zero: plain means over all tokens, so it only contributes zeros"""
    _split(monkeypatch, True, 1003, torch.float32)
    d = gpu_case(torch.float32, 4, 75, 64, 1003, zero_row=True)
    compare(kind, d, (None, 'k3', True))


@gpu
@pytest.mark.parametrize('kind,needs', [('ppo', (True, False)), ('ppo', (False, True)), ('a2c', (True, False, False)),
                                        ('a2c', (False, True, False)), ('a2c', (False, False, True))])
@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
def test_one_input_requires_grad(monkeypatch, kind, needs, dtype):
    _split(monkeypatch, True, 32771, torch.float32)
    compare(kind, gpu_case(dtype, 4, 75, 64, 32771), (2.0, 'k3', True), needs)


@gpu
@pytest.mark.parametrize('kind', ['ppo', 'a2c'])
def test_tied_weight(monkeypatch, kind):
    """hidden built from the lm_head's own embedding: autograd adds both gradients"""
    _split(monkeypatch, True, 1003, torch.float32)
    d = gpu_case(torch.float32, 4, 75, 64, 1003)
    tokens = torch.randint(0, 1003, (4, 75), device='cuda')
    res = []
    for form in ('linear', 'logits'):
        emb = d['lm_weight'].detach().clone().requires_grad_(True)
        h = torch.tanh(F.embedding(tokens, emb) * 3 + d['hidden'])
        if kind == 'ppo':
            if form == 'linear':
                loss = ppo_call(dict(d, hidden=h, lm_weight=emb), kl_type='k3', entropy_weight=EW, kl_weight=KW)[0].loss
            else:
                p, _ = R.ppo_policy_error(R.ppo_policy_data(F.linear(h, emb), d['logit_old'], d['action'], d['adv'],
                                                            d['weight'], d['logit_pretrained']), kl_type='k3')
                loss = p.policy_loss - EW * p.entropy_loss + KW * p.kl_div
        else:
            if form == 'linear':
                loss = a2c_call(dict(d, hidden=h, lm_weight=emb), value_weight=VW, entropy_weight=EW).loss
            else:
                a = R.a2c_error(R.a2c_data(F.linear(h, emb), d['action'], d['value'], d['adv'], d['return_'],
                                           d['weight']))
                loss = a.policy_loss + VW * a.value_loss - EW * a.entropy_loss
        loss.backward()
        res.append((loss.item(), emb.grad))
    np.testing.assert_allclose(res[0][0], res[1][0], rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(res[0][1], res[1][1], rtol=1e-5, atol=1e-5 * float(res[1][1].abs().max()))


@gpu
@pytest.mark.parametrize('kind', ['ppo', 'a2c'])
@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
def test_upstream_gradient_not_one(monkeypatch, kind, dtype):
    """0.5 * loss + another term, and a second backward through the same graph"""
    _split(monkeypatch, True, 1003, torch.float32)
    d = gpu_case(dtype, 4, 75, 64, 1003)
    grads = []
    for form in ('linear', 'logits'):
        h, w, v = _leaves(d, (True, True, True))
        if kind == 'ppo':
            if form == 'linear':
                loss = ppo_call(dict(d, hidden=h, lm_weight=w), kl_type='k3', entropy_weight=EW, kl_weight=KW)[0].loss
            else:
                p, _ = R.ppo_policy_error(R.ppo_policy_data(F.linear(h, w), d['logit_old'], d['action'], d['adv'],
                                                            d['weight'], d['logit_pretrained']), kl_type='k3')
                loss = p.policy_loss - EW * p.entropy_loss + KW * p.kl_div
        else:
            if form == 'linear':
                loss = a2c_call(dict(d, hidden=h, lm_weight=w, value=v), value_weight=VW, entropy_weight=EW).loss
            else:
                a = R.a2c_error(R.a2c_data(F.linear(h, w), d['action'], v, d['adv'], d['return_'], d['weight']))
                loss = a.policy_loss + VW * a.value_loss - EW * a.entropy_loss
        total = 0.5 * loss + (h.float() ** 2).mean() + w.float().sum() * 1e-3 + (v ** 2).mean()
        total.backward(retain_graph=True)
        first = (h.grad.clone(), w.grad.clone(), v.grad.clone())
        h.grad = w.grad = v.grad = None
        (3.0 * loss).backward()
        second = (h.grad, w.grad, v.grad if kind == 'a2c' else torch.zeros(()))
        grads.append(first + second)
    for got, comp in zip(*grads):
        rtol = 1e-5 if dtype == torch.float32 else 2 ** -6
        torch.testing.assert_close(got.float(), comp.float(), rtol=rtol, atol=rtol * float(comp.float().abs().max()))


@gpu
@pytest.mark.parametrize('kind', ['ppo', 'a2c'])
def test_bit_identical_repeats(monkeypatch, kind):
    _split(monkeypatch, True, 32771, torch.bfloat16)
    d = gpu_case(torch.bfloat16, 4, 75, 64, 32771)
    a, b = ours(kind, d, (2.0, 'k3', True)), ours(kind, d, (2.0, 'k3', True))
    assert a[0] == b[0]
    for k in (1, 2, 3):
        assert (a[k] is None and b[k] is None) or torch.equal(a[k], b[k])


@gpu
@pytest.mark.parametrize('kind', ['ppo', 'a2c'])
def test_peak_memory(kind):
    """(8, 1024, 1024, 152 064) bf16: forward + backward stays within the chunk buffer + the fp32 dW accumulator + dW +
    dH + O(B*S), and below half of what F.linear + the logit-form loss allocates"""
    B, S, D, V = 8, 1024, 1024, 152064
    d = gpu_case(torch.bfloat16, B, S, D, V, mask=True)
    N = B * S
    rows, _ = ops.lm_chunk_plan(N, V, 2, ops.sm_count(torch.device('cuda')), True, 5 if kind == 'ppo' else 3)
    slack = 64 * N * 4 + (8 << 20)  # O(B*S) per-row buffers, allocator rounding

    def peak(fn):
        h, w, v = _leaves(d, (True, True, True))
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        fn(h, w, v)
        torch.cuda.synchronize()
        return torch.cuda.max_memory_allocated() - base

    def linear(h, w, v):
        if kind == 'ppo':
            loss = ppo_call(dict(d, hidden=h, lm_weight=w), kl_type='k3', entropy_weight=EW, kl_weight=KW)[0].loss
        else:
            loss = a2c_call(dict(d, hidden=h, lm_weight=w, value=v), value_weight=VW, entropy_weight=EW).loss
        loss.backward()

    def logits(h, w, v):
        if kind == 'ppo':
            p, _ = R.ppo_policy_error(R.ppo_policy_data(F.linear(h, w), d['logit_old'], d['action'], d['adv'],
                                                        d['weight'], d['logit_pretrained']), kl_type='k3')
            loss = p.policy_loss - EW * p.entropy_loss + KW * p.kl_div
        else:
            a = R.a2c_error(R.a2c_data(F.linear(h, w), d['action'], v, d['adv'], d['return_'], d['weight']))
            loss = a.policy_loss + VW * a.value_loss - EW * a.entropy_loss
        loss.backward()

    ours_b, comp_b = peak(linear), peak(logits)
    bound = rows * V * 2 + V * D * 4 + V * D * 2 + N * D * 2 + slack  # chunk, dW accumulator, dW, dH
    assert ours_b <= bound, (ours_b, bound)
    assert ours_b < comp_b / 2, (ours_b, comp_b)


@gpu
@pytest.mark.parametrize('kind', ['ppo', 'a2c'])
@pytest.mark.parametrize('backend', ['aot_eager', 'inductor'])
def test_compile_learner_step(monkeypatch, kind, backend):
    """torch.compile(fullgraph=False) around a step that calls the loss: it runs eagerly behind a graph break and the step
    gives the eager result -- bit for bit under aot_eager, within 1e-5 of the largest entry under inductor"""
    _split(monkeypatch, True, 1003, torch.float32)
    d = gpu_case(torch.float32, 4, 75, 64, 1003)
    torch.manual_seed(1)
    layer = torch.nn.Linear(64, 64).cuda()
    head = torch.nn.Linear(64, 1).cuda()

    def step(x, w):
        h = torch.tanh(layer(x))
        if kind == 'ppo':
            loss, _ = ppo_call(dict(d, hidden=h, lm_weight=w), kl_type='k3', entropy_weight=EW, kl_weight=KW)
            value = head(h).squeeze(-1)
            vl = R.ppo_value_error(R.ppo_value_data(value, d['value'], d['return_'], d['weight']), 0.2, True)
            return loss.loss + VW * vl
        loss = a2c_call(dict(d, hidden=h, lm_weight=w, value=head(h).squeeze(-1)), value_weight=VW, entropy_weight=EW)
        return loss.loss * 2.0

    torch._dynamo.reset()
    res = []
    for fn in (step, torch.compile(step, backend=backend, fullgraph=False)):
        layer.zero_grad()
        head.zero_grad()
        w = d['lm_weight'].detach().clone().requires_grad_(True)
        loss = fn(d['hidden'], w)
        loss.backward()
        res.append((loss.detach(), w.grad, layer.weight.grad.clone(), head.weight.grad.clone()))
    for a, b in zip(*res):
        if backend == 'aot_eager':
            assert torch.equal(a, b), float((a - b).abs().max())
        else:
            err, scale = float((a - b).abs().max()), float(b.abs().max())
            assert err <= 1e-5 * scale, (err, scale)
