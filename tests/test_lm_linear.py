"""grpo_policy_error_linear, rloo_policy_error_linear and token_logp_linear (rl_utils/lm_linear.py): the losses from the
lm_head's hidden states, the logits one chunk of token rows at a time.

CPU, on a recording stand-in for the CUDA library: argument checks, the chunk plan (rows per chunk, a sequence split
across a chunk boundary, the capacity of the loss partials), the autograd wiring (only the inputs that require grad get
gradient GEMMs) and that no (B*S, V) tensor is ever allocated.

GPU: loss, approx_kl, clipfrac, d hidden and d lm_weight against the library's own composition (F.linear + the logit
losses) and against a float64 restatement (tests/grpo_oracle.py).  fp32: the LM tests' 1e-5 rule.  bf16: max|ours -
fp64| <= 2 * max|composition - fp64| + 1e-6 * max|fp64|, since the chunked GEMMs may round differently from one large
GEMM.  Also: an all-zero mask row, each input alone requiring grad, a tied weight, an upstream gradient != 1,
determinism, peak memory and torch.compile."""
import contextlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from torch.utils._python_dispatch import TorchDispatchMode

import di_engine_b200 as b2
from di_engine_b200 import _lib, ops
from tests import grpo_oracle as go

R = b2.rl_utils


# ----------------------------------------------------------------------------------------------------------------
# CPU: the recording stand-in
# ----------------------------------------------------------------------------------------------------------------
class _RecordingLib:
    """checks every call against the ctypes prototypes and records (name, args)"""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        proto = _lib.PROTOTYPES[name]

        def fn(*args):
            assert len(args) == len(proto), (name, len(args), len(proto))
            for a, ty in zip(args, proto):
                ty.from_param(a)
            self.calls.append((name, args))
            return 0

        if name == 'b200rl_workspace_bytes':
            return lambda: 1 << 20
        return fn

    def names(self):
        return [c[0] for c in self.calls]


@pytest.fixture
def dry(monkeypatch):
    rec = _RecordingLib()
    monkeypatch.setattr(ops, 'lib', lambda: rec)
    monkeypatch.setattr(ops, 'require_cuda', lambda: None)
    monkeypatch.setattr(ops, 'compute_device', lambda *t: torch.device('cpu'))
    monkeypatch.setattr(ops, 'stream_ptr', lambda: 0)
    monkeypatch.setattr(ops, 'sm_count', lambda dev: 132)
    monkeypatch.setattr(torch.cuda, 'device', lambda d: contextlib.nullcontext())
    ops._WS.clear()
    yield rec
    ops._WS.clear()


class _Ops(TorchDispatchMode):
    """the aten ops of a call and the shapes of the tensors they return"""

    def __init__(self):
        super().__init__()
        self.ops = []

    def __torch_dispatch__(self, func, types, args=(), kwargs=None):
        out = func(*args, **(kwargs or {}))
        outs = out if isinstance(out, (tuple, list)) else (out, )
        self.ops.append((func.overloadpacket.__name__, [tuple(o.shape) for o in outs if isinstance(o, torch.Tensor)]))
        return out

    def count(self, *names):
        return sum(1 for n, _ in self.ops if n in names)

    def allocated(self):
        return [s for n, shapes in self.ops if n.startswith(('empty', 'zeros', 'new_empty')) for s in shapes]


B_, S_, D_, V_ = 3, 100, 8, 1031  # 300 rows: chunks of 128, 128 and 44 rows when the budget holds 128 rows


def make(kind='grpo', dtype=torch.float32, B=B_, S=S_, D=D_, V=V_, weight=True, seed=0, device='cpu'):
    g = torch.Generator().manual_seed(seed)
    h = torch.randn(B, S, D, generator=g).to(dtype)
    w = (torch.randn(V, D, generator=g) / D ** 0.5).to(dtype)
    d = {
        'hidden': h, 'lm_weight': w,
        'action': torch.randint(0, V, (B, S), generator=g),
        'logp_old': -torch.rand(B, S, generator=g) * 6 - 1,
        'logp_ref': -torch.rand(B, S, generator=g) * 6 - 1,
        'adv': torch.randn(B, generator=g),
        'reward': torch.randn(B, 1, generator=g) if kind == 'rloo' else None,  # K = B groups of one prompt
        'weight': (torch.rand(B, S, generator=g) > 0.2).float() if weight else None,
    }
    return {k: (v.to(device) if isinstance(v, torch.Tensor) else v) for k, v in d.items()}


def loss_call(kind, d, **kw):
    if kind == 'grpo':
        return R.grpo_policy_error_linear(R.grpo_linear_data(d['hidden'], d['lm_weight'], d['logp_old'], d['logp_ref'],
                                                             d['action'], d['adv'], d['weight']), **kw)
    return R.rloo_policy_error_linear(R.rloo_linear_data(d['hidden'], d['lm_weight'], d['logp_old'], d['action'],
                                                         d['reward'], d['weight']), **kw)


@pytest.fixture
def rows128(monkeypatch):
    monkeypatch.setattr(ops, 'LM_CHUNK_BYTES', 128 * V_ * 4)


@pytest.mark.filterwarnings('ignore:invalid value encountered in cast')  # the stand-in leaves outputs uninitialised
@pytest.mark.parametrize('kind', ['grpo', 'rloo'])
@pytest.mark.parametrize('grads', [(True, True), (True, False), (False, True), (False, False)])
def test_loss_wiring_and_chunks(dry, rows128, kind, grads):
    """one row launch per chunk at rows [0, 128), [128, 256), [256, 300) -- the sequence b = 1 (rows 100..199) straddles a
    boundary; a dH GEMM per chunk only if hidden requires grad, a dW GEMM only if lm_weight does; an in-place scale of
    each at backward; and never a (B*S, V) tensor"""
    d = make(kind)
    d['hidden'].requires_grad_(grads[0])
    d['lm_weight'].requires_grad_(grads[1])
    with _Ops() as rec:
        loss, info = loss_call(kind, d)
        if any(grads):
            loss.backward()
    fwd = [c for c in dry.calls if c[0] == 'b200rl_lm_linear_fwd']
    assert [(c[1][3], c[1][4], c[1][5]) for c in fwd] == [(0, 128, 128), (128, 128, 128), (256, 44, 128)]
    assert all(c[1][0] == (0 if kind == 'grpo' else 1) and c[1][22] == int(any(grads)) for c in fwd)
    assert all(c[1][16] == fwd[0][1][16] for c in fwd)  # one sequence-normaliser buffer for the whole call
    assert dry.names()[3:] == ['b200rl_lm_linear_scale'] * sum(grads)
    assert rec.count('mm') == 3 + 3 * grads[0]
    assert rec.count('addmm', 'addmm_') == 3 * grads[1]
    assert all(int(np.prod(s)) < B_ * S_ * V_ for s in rec.allocated())
    assert sum(1 for s in rec.allocated() if s == (128, V_)) == 1  # one chunk buffer per call
    assert isinstance(info.approx_kl, float) and isinstance(info.clipfrac, float)
    if grads[0]:
        assert d['hidden'].grad.shape == d['hidden'].shape and d['hidden'].grad.dtype == torch.float32
    if grads[1]:
        assert d['lm_weight'].grad.shape == (V_, D_)
    if not any(grads):
        assert (B_ * S_, D_) not in rec.allocated() and (V_, D_) not in rec.allocated()


@pytest.mark.filterwarnings('ignore:invalid value encountered in cast')
def test_token_logp_wiring(dry, rows128):
    d = make()
    d['hidden'].requires_grad_(True)
    d['lm_weight'].requires_grad_(True)
    with _Ops() as rec:
        lp = R.token_logp_linear(d['hidden'], d['lm_weight'], d['action'])
    assert lp.shape == (B_, S_) and lp.dtype == torch.float32
    assert dry.names() == ['b200rl_lm_linear_fwd'] * 3 and rec.count('mm') == 3
    assert all(c[1][0] == 2 for c in dry.calls)
    with _Ops() as rec:
        lp.backward(torch.randn(B_, S_))
    bwd = [c for c in dry.calls if c[0] == 'b200rl_lm_linear_bwd']
    assert [(c[1][2], c[1][3]) for c in bwd] == [(0, 128), (128, 128), (256, 44)]
    # the logit GEMM again, dH and dW per chunk
    assert rec.count('mm') == 6 and rec.count('addmm', 'addmm_') == 3
    assert d['hidden'].grad.shape == d['hidden'].shape and d['lm_weight'].grad.shape == (V_, D_)


@pytest.mark.filterwarnings('ignore:invalid value encountered in cast')
def test_token_logp_no_grad_allocates_no_gradient_buffer(dry, rows128):
    d = make()
    d['hidden'].requires_grad_(True)
    d['lm_weight'].requires_grad_(True)
    with torch.no_grad(), _Ops() as rec:
        lp = R.token_logp_linear(d['hidden'], d['lm_weight'], d['action'])
    assert not lp.requires_grad
    assert sorted(rec.allocated()) == sorted([(128, V_), (B_ * S_, ), (B_ * S_, )])  # chunk, lp, lse


def test_chunk_plan(monkeypatch):
    monkeypatch.setattr(ops, 'LM_CHUNK_BYTES', 512 << 20)
    # Qwen2-7B's vocabulary in bf16: 1664 rows (a multiple of 128) of 304 KB each
    assert ops.lm_chunk_plan(16 * 1024, 152064, 2, 132, True) == (1664, 10)
    assert ops.lm_chunk_plan(100, 152064, 2, 132, True) == (100, 1)  # fewer rows than a chunk: all of them
    assert ops.lm_chunk_plan(16 * 1024, 32768, 4, 132, True) == (4096, 4)
    monkeypatch.setattr(ops, 'LM_CHUNK_BYTES', 1)
    assert ops.lm_chunk_plan(1000, 50, 4, 132, False) == (128, 8)  # never fewer than 128 rows
    # 128-row chunks: 128 CTAs x 3 partials each; 666 chunks fit below the workspace's 256 000 partial words, 667 do not
    assert ops.lm_chunk_plan(666 * 128, 50, 4, 132, True) == (128, 666)
    with pytest.raises(ValueError, match='partials'):
        ops.lm_chunk_plan(667 * 128, 50, 4, 132, True)
    assert ops.lm_chunk_plan(667 * 128, 50, 4, 132, False) == (128, 667)  # the log-prob mode stores none


def test_partials_overflow_raises_before_any_launch(dry, monkeypatch):
    monkeypatch.setattr(ops, 'LM_CHUNK_BYTES', 1)
    d = make(B=2, S=667 * 64, D=2, V=3, weight=False)
    with pytest.raises(ValueError, match='partials'):
        loss_call('grpo', d)
    assert dry.calls == []


@pytest.mark.parametrize('dtype', [torch.float16, torch.float64])
def test_other_dtypes_raise(dry, dtype):
    d = make()
    d['hidden'], d['lm_weight'] = d['hidden'].to(dtype), d['lm_weight'].to(dtype)
    with pytest.raises(TypeError, match='float32 or both bfloat16'):
        loss_call('grpo', d)
    with pytest.raises(TypeError, match='float32 or both bfloat16'):
        R.token_logp_linear(d['hidden'], d['lm_weight'], d['action'])


def test_mixed_dtypes_raise(dry):
    d = make()
    d['lm_weight'] = d['lm_weight'].bfloat16()
    with pytest.raises(TypeError, match='both'):
        loss_call('rloo', make('rloo') | {'lm_weight': d['lm_weight']})


@pytest.mark.filterwarnings('ignore:invalid value encountered in cast')
def test_side_inputs_of_any_float_dtype_are_read_as_fp32(dry):
    d = make()
    for k in ('logp_old', 'logp_ref', 'weight'):
        d[k] = d[k].double()
    d['adv'] = d['adv'].bfloat16()
    loss_call('grpo', d)
    assert dry.names() == ['b200rl_lm_linear_fwd']


@pytest.mark.parametrize('field,value,err', [
    ('hidden', torch.zeros(300, 8), 'hidden must be'),
    ('lm_weight', torch.zeros(1031, 9), 'lm_weight must be'),
    ('lm_weight', torch.zeros(1031), 'lm_weight must be'),
    ('action', torch.zeros(3, 99, dtype=torch.long), 'action must be'),
    ('weight', torch.ones(3, 101), 'weight must be'),
    ('adv', torch.zeros(4), 'adv must'),
    ('logp_old', torch.zeros(3, 99), 'logp_old must be'),
    ('logp_ref', torch.zeros(300), 'logp_ref must be'),
])
def test_argument_errors(dry, field, value, err):
    d = make()
    d[field] = value
    with pytest.raises(RuntimeError, match=err):
        loss_call('grpo', d)
    assert dry.calls == []


def test_token_logp_argument_errors(dry):
    d = make()
    with pytest.raises(RuntimeError, match='index must be'):
        R.token_logp_linear(d['hidden'], d['lm_weight'], d['action'][:, :-1])
    with pytest.raises(RuntimeError, match='lm_weight must be'):
        R.token_logp_linear(d['hidden'], d['lm_weight'][:, :-1], d['action'])


def test_out_of_range_action_raises_with_index_checks(dry, monkeypatch):
    monkeypatch.setattr(ops, 'CHECK_INDICES', True)
    d = make()
    d['action'][1, 7] = V_
    with pytest.raises(IndexError, match='out of range'):
        loss_call('grpo', d)
    with pytest.raises(IndexError, match='out of range'):
        R.token_logp_linear(d['hidden'], d['lm_weight'], d['action'])
    assert dry.calls == []


def test_exports_stay_outside_the_reference_lists():
    for name in ('token_logp_linear', 'grpo_policy_error_linear', 'rloo_policy_error_linear'):
        assert callable(getattr(R, name))
        assert name not in R.HOT_PATH_FUNCTIONS and name not in R.LM_HOT_PATH_FUNCTIONS


# ----------------------------------------------------------------------------------------------------------------
# GPU
# ----------------------------------------------------------------------------------------------------------------
gpu = pytest.mark.gpu


def gpu_case(kind, dtype, B, S, D, V, seed=0, mask=True, zero_row=False):
    """hidden / lm_weight on the device, and logp_old / logp_ref from perturbed hidden states of the same head (so the
    ratios sit around 1 and some clip); the logit tensors of the composition are kept for it"""
    torch.manual_seed(seed)
    dev = torch.device('cuda')
    h = (torch.randn(B, S, D, device=dev) * 2).to(dtype)
    w = torch.randn(V, D, device=dev).div(D ** 0.5).to(dtype)
    action = torch.randint(0, V, (B, S), device=dev)
    h_old = (h.float() + 0.05 * torch.randn_like(h.float())).to(dtype)
    h_ref = (h.float() + 0.05 * torch.randn_like(h.float())).to(dtype)
    with torch.no_grad():
        logit_old, logit_ref = F.linear(h_old, w), F.linear(h_ref, w)
        lp_old, lp_ref = R.efficient_method(logit_old, action), R.efficient_method(logit_ref, action)
    weight = (torch.rand(B, S, device=dev) > 0.25).float() if mask else None
    if zero_row:
        weight[1] = 0
    d = {'hidden': h, 'lm_weight': w, 'action': action, 'logp_old': lp_old, 'logp_ref': lp_ref,
         'logit_old': logit_old, 'logit_ref': logit_ref, 'weight': weight,
         'adv': torch.randn(B, device=dev), 'reward': torch.randn(2, B // 2, device=dev) if kind == 'rloo' else None}
    return d


def composition(kind, d, needs=(True, True)):
    """F.linear + the library's logit losses: loss, approx_kl, clipfrac, d hidden, d lm_weight"""
    h = d['hidden'].detach().clone().requires_grad_(needs[0])
    w = d['lm_weight'].detach().clone().requires_grad_(needs[1])
    logits = F.linear(h, w)
    if kind == 'grpo':
        loss, info = R.grpo_policy_error(R.grpo_policy_data(logits, d['logit_old'], d['logit_ref'], d['action'],
                                                            d['adv'], d['weight']), R.efficient_method, go.CLIP, go.BETA)
    else:
        loss, info = R.rloo_policy_error(R.rloo_policy_data(logits, d['logit_old'], d['action'], d['reward'],
                                                            d['weight']), R.efficient_method, go.CLIP)
    loss.backward()
    return loss.item(), info.approx_kl, info.clipfrac, h.grad, w.grad


def ours(kind, d, needs=(True, True)):
    h = d['hidden'].detach().clone().requires_grad_(needs[0])
    w = d['lm_weight'].detach().clone().requires_grad_(needs[1])
    loss, info = loss_call(kind, dict(d, hidden=h, lm_weight=w), clip_ratio=go.CLIP, **({'beta': go.BETA} if kind == 'grpo' else {}))
    loss.backward()
    return loss.item(), info.approx_kl, info.clipfrac, h.grad, w.grad


def fp64(kind, d):
    """the float64 restatement: loss, approx_kl, clipfrac, d hidden, d lm_weight"""
    h = d['hidden'].double().requires_grad_(True)
    w = d['lm_weight'].double().requires_grad_(True)
    logits = h @ w.t()
    lp_new = go.logp64(logits, d['action'])
    adv = d['adv'] if kind == 'grpo' else go.rloo_adv64(d['reward'])
    loss, kl, cf = go.head64(lp_new, d['logp_old'].double(), d['logp_ref'].double() if kind == 'grpo' else None,
                             adv.double(), d['weight'], go.CLIP, go.BETA if kind == 'grpo' else 0.0)
    loss.backward()
    return loss.item(), kl.item(), cf.item(), h.grad, w.grad


def check_scalar(got, comp, want, bf16, slack=0.0):
    """slack: clipfrac may count a token more or less where a ratio sits within rounding of a clip bound"""
    if bf16:
        assert abs(got - want) <= 2 * abs(comp - want) + 1e-6 * abs(want) + slack, (got, comp, want)
    else:
        np.testing.assert_allclose(got, want, rtol=1e-5, atol=1e-5 * max(1.0, abs(want)) + slack)


def check_tensor(got, comp, want, bf16):
    """bf16: max|ours - fp64| <= 2 max|composition - fp64| + 1e-6 max|fp64|; fp32: the 1e-5 rule of tests/test_grpo_rloo"""
    got, comp, want = got.double(), comp.double(), want.double().to(got.device)
    assert torch.equal(torch.isnan(got), torch.isnan(want))
    fin = ~torch.isnan(want)
    got, comp, want = got[fin], comp[fin], want[fin]
    scale = float(want.abs().max()) if want.numel() else 0.0
    err = float((got - want).abs().max()) if want.numel() else 0.0
    comp_err = float((comp - want).abs().max()) if want.numel() else 0.0
    if bf16:
        assert err <= 2 * comp_err + 1e-6 * scale, (err, comp_err, scale)
    else:  # 1e-5 of the largest entry (or, under a TF32 matmul setting, the composition's own error rule)
        assert err <= max(1e-5 * scale, 2 * comp_err + 1e-6 * scale), (err, comp_err, scale)


def compare(kind, d, needs=(True, True)):
    bf16 = d['hidden'].dtype == torch.bfloat16
    got, comp, want = ours(kind, d, needs), composition(kind, d, needs), fp64(kind, d)
    N = d['action'].numel()
    for k in range(3):
        check_scalar(got[k], comp[k], want[k], bf16, 2.0 / N if k == 2 else 0.0)
    for k, need in zip((3, 4), needs):
        if need:
            check_tensor(got[k], comp[k], want[k], bf16)
        else:
            assert got[k] is None
    return got


@gpu
@pytest.mark.parametrize('kind', ['grpo', 'rloo'])
@pytest.mark.parametrize('dtype,V', [(torch.float32, 1003), (torch.bfloat16, 1003), (torch.float32, 32771),
                                     (torch.bfloat16, 32771), (torch.bfloat16, 152064)])
@pytest.mark.parametrize('split', [False, True])
def test_against_composition_and_fp64(monkeypatch, kind, dtype, V, split):
    """split: 128-row chunks over 4 x 75 tokens -- 300 is no multiple of the chunk, and sequences 1 and 3 straddle
    boundaries"""
    if split:
        monkeypatch.setattr(ops, 'LM_CHUNK_BYTES', 128 * V * torch.tensor([], dtype=dtype).element_size())
    compare(kind, gpu_case(kind, dtype, 4, 75, 64, V))


@gpu
@pytest.mark.parametrize('kind', ['grpo', 'rloo'])
def test_all_zero_mask_row(monkeypatch, kind):
    """a sequence whose weights sum to 0: NaN loss, as the reference"""
    monkeypatch.setattr(ops, 'LM_CHUNK_BYTES', 128 * 1003 * 4)
    d = gpu_case(kind, torch.float32, 4, 75, 64, 1003, zero_row=True)
    got, comp = ours(kind, d), composition(kind, d)
    assert np.isnan(got[0]) and np.isnan(comp[0])
    for k in (3, 4):
        assert torch.equal(torch.isnan(got[k]), torch.isnan(comp[k]))


@gpu
@pytest.mark.parametrize('needs', [(True, False), (False, True)])
@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
def test_one_input_requires_grad(monkeypatch, needs, dtype):
    monkeypatch.setattr(ops, 'LM_CHUNK_BYTES', 128 * 32771 * 4)
    compare('grpo', gpu_case('grpo', dtype, 4, 75, 64, 32771), needs)


@gpu
def test_tied_weight(monkeypatch):
    """hidden built from the lm_head's own embedding: autograd adds both gradients"""
    monkeypatch.setattr(ops, 'LM_CHUNK_BYTES', 128 * 1003 * 4)
    d = gpu_case('grpo', torch.float32, 4, 75, 64, 1003)
    tokens = torch.randint(0, 1003, (4, 75), device='cuda')

    def run(fn):
        emb = d['lm_weight'].detach().clone().requires_grad_(True)
        h = torch.tanh(F.embedding(tokens, emb) * 3 + d['hidden'])
        loss, _ = fn(h, emb)
        loss.backward()
        return loss.item(), emb.grad

    l1, g1 = run(lambda h, e: R.grpo_policy_error_linear(R.grpo_linear_data(
        h, e, d['logp_old'], d['logp_ref'], d['action'], d['adv'], d['weight'])))
    l2, g2 = run(lambda h, e: R.grpo_policy_error(R.grpo_policy_data(
        F.linear(h, e), d['logit_old'], d['logit_ref'], d['action'], d['adv'], d['weight'])))
    np.testing.assert_allclose(l1, l2, rtol=1e-5)
    torch.testing.assert_close(g1, g2, rtol=1e-5, atol=1e-5 * float(g2.abs().max()))


@gpu
@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
def test_upstream_gradient_not_one(monkeypatch, dtype):
    """0.5 * loss + another term, and a second backward through the same graph"""
    monkeypatch.setattr(ops, 'LM_CHUNK_BYTES', 128 * 1003 * 4)
    d = gpu_case('grpo', dtype, 4, 75, 64, 1003)
    grads = []
    for fn in ('linear', 'logits'):
        h = d['hidden'].detach().clone().requires_grad_(True)
        w = d['lm_weight'].detach().clone().requires_grad_(True)
        if fn == 'linear':
            loss, _ = R.grpo_policy_error_linear(R.grpo_linear_data(h, w, d['logp_old'], d['logp_ref'], d['action'],
                                                                    d['adv'], d['weight']))
        else:
            loss, _ = R.grpo_policy_error(R.grpo_policy_data(F.linear(h, w), d['logit_old'], d['logit_ref'], d['action'],
                                                             d['adv'], d['weight']))
        total = 0.5 * loss + (h.float() ** 2).mean() + w.float().sum() * 1e-3
        total.backward(retain_graph=True)
        first = (h.grad.clone(), w.grad.clone())
        h.grad = w.grad = None
        (3.0 * loss).backward()
        grads.append(first + (h.grad, w.grad))
    for got, comp in zip(*grads):
        rtol = 1e-5 if dtype == torch.float32 else 2 ** -6
        torch.testing.assert_close(got.float(), comp.float(), rtol=rtol, atol=rtol * float(comp.float().abs().max()))


@gpu
@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
def test_token_logp_linear(monkeypatch, dtype):
    monkeypatch.setattr(ops, 'LM_CHUNK_BYTES', 128 * 32771 * 4)
    d = gpu_case('grpo', dtype, 4, 75, 64, 32771)
    g = torch.randn(4, 75, device='cuda')
    res = []
    for fn in ('linear', 'logits', 'fp64'):
        h = d['hidden'].detach().clone().requires_grad_(True)
        w = d['lm_weight'].detach().clone().requires_grad_(True)
        if fn == 'linear':
            lp = R.token_logp_linear(h, w, d['action'])
        elif fn == 'logits':
            lp = R.efficient_method(F.linear(h, w), d['action'])
        else:
            h, w = h.detach().double().requires_grad_(True), w.detach().double().requires_grad_(True)
            lp = go.logp64(h @ w.t(), d['action'])
        (lp * g.to(lp.dtype)).sum().backward()
        res.append((lp.detach(), h.grad, w.grad))
    bf16 = dtype == torch.bfloat16
    for k in range(3):
        check_tensor(res[0][k], res[1][k], res[2][k], bf16)
    with torch.no_grad():
        lp = R.token_logp_linear(d['hidden'], d['lm_weight'], d['action'])
    assert torch.equal(lp, res[0][0])


@gpu
@pytest.mark.parametrize('kind', ['grpo', 'rloo'])
def test_bit_identical_repeats(monkeypatch, kind):
    monkeypatch.setattr(ops, 'LM_CHUNK_BYTES', 128 * 32771 * 2)
    d = gpu_case(kind, torch.bfloat16, 4, 75, 64, 32771)
    a, b = ours(kind, d), ours(kind, d)
    assert a[:3] == b[:3]
    assert torch.equal(a[3], b[3]) and torch.equal(a[4], b[4])


@gpu
def test_peak_memory():
    """(8, 1024, 1024, 152 064) bf16: forward + backward stays within the chunk buffer + the fp32 dW accumulator + dH
    + O(B*S), and below half of what F.linear + grpo_policy_error allocates; the no_grad log-prob call holds the chunk
    buffer and O(B*S) only"""
    B, S, D, V = 8, 1024, 1024, 152064
    d = gpu_case('grpo', torch.bfloat16, B, S, D, V, mask=True)
    N = B * S
    rows, _ = ops.lm_chunk_plan(N, V, 2, ops.sm_count(torch.device('cuda')), True)
    slack = 64 * N * 4 + (8 << 20)  # O(B*S) per-row buffers, allocator rounding

    def peak(fn):
        h = d['hidden'].detach().clone().requires_grad_(True)
        w = d['lm_weight'].detach().clone().requires_grad_(True)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        fn(h, w)
        torch.cuda.synchronize()
        return torch.cuda.max_memory_allocated() - base

    def linear(h, w):
        loss, _ = R.grpo_policy_error_linear(R.grpo_linear_data(h, w, d['logp_old'], d['logp_ref'], d['action'],
                                                                d['adv'], d['weight']))
        loss.backward()

    def logits(h, w):
        loss, _ = R.grpo_policy_error(R.grpo_policy_data(F.linear(h, w), d['logit_old'], d['logit_ref'], d['action'],
                                                         d['adv'], d['weight']))
        loss.backward()

    ours_b, comp_b = peak(linear), peak(logits)
    bound = rows * V * 2 + V * D * 4 + V * D * 2 + N * D * 2 + slack  # chunk, dW accumulator, dW, dH
    assert ours_b <= bound, (ours_b, bound)
    assert ours_b < comp_b / 2, (ours_b, comp_b)
    with torch.no_grad():
        nog = peak(lambda h, w: R.token_logp_linear(h, w, d['action']))
    assert nog <= rows * V * 2 + slack, nog


@gpu
@pytest.mark.parametrize('backend', ['aot_eager', 'inductor'])
def test_compile_learner_step(monkeypatch, backend):
    """torch.compile(fullgraph=False) around a step that calls grpo_policy_error_linear: the loss runs eagerly behind a
    graph break and the step gives the eager result -- bit for bit where the compiled parts run torch's own kernels
    (aot_eager), within 1e-5 of the largest entry where inductor writes its own (the tanh of the layer before)"""
    monkeypatch.setattr(ops, 'LM_CHUNK_BYTES', 128 * 1003 * 4)
    d = gpu_case('grpo', torch.float32, 4, 75, 64, 1003)
    torch.manual_seed(1)
    layer = torch.nn.Linear(64, 64).cuda()

    def step(x, w):
        h = torch.tanh(layer(x))
        loss, info = R.grpo_policy_error_linear(R.grpo_linear_data(h, w, d['logp_old'], d['logp_ref'], d['action'],
                                                                   d['adv'], d['weight']))
        return loss * 2.0

    torch._dynamo.reset()
    res = []
    for fn in (step, torch.compile(step, backend=backend, fullgraph=False)):
        layer.zero_grad()
        w = d['lm_weight'].detach().clone().requires_grad_(True)
        loss = fn(d['hidden'], w)
        loss.backward()
        res.append((loss.detach(), w.grad, layer.weight.grad.clone()))
    for a, b in zip(*res):
        if backend == 'aot_eager':
            assert torch.equal(a, b), float((a - b).abs().max())
        else:
            err, scale = float((a - b).abs().max()), float(b.abs().max())
            assert err <= 1e-5 * scale, (err, scale)
