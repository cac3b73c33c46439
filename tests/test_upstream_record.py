"""The verify launch of the forward-written gradients (include/b200rl.h) when no record is passed.

A repeated backward through one graph gets fresh gradient buffers and no record of the upstream gradients the forward
launch used, so its verify launch must recompute.  With all-NaN upstream gradients every gradient is NaN; the free blocks of
the caching allocator are filled with a finite sentinel first, so a launch that skipped would hand that sentinel to autograd.
"""
import numpy as np
import pytest
import torch

import di_engine_b200 as b2
from di_engine_b200 import ops
from oracle import rl_oracle
from tests import cases
from tests import ppo_lm_oracle as po

pytestmark = pytest.mark.gpu
DEV = 'cuda'
SENTINEL = 3.0


@pytest.fixture(autouse=True)
def keep_records():
    """NaN upstream gradients refresh the call sites' records: put them back for the tests that follow"""
    saved = {k: v.clone() for k, v in ops._HINT.items()}
    yield
    for k, v in ops._HINT.items():
        v.copy_(saved[k] if k in saved else torch.tensor(ops._HINT_INIT[k[1]]))


def fill_free_blocks():
    """Allocate every free block of the caching allocator (largest first, so each request takes a block of its own size),
    fill it with SENTINEL and free it again."""
    torch.cuda.synchronize()
    sizes = sorted((b['size'] for s in torch.cuda.memory_snapshot() for b in s['blocks'] if b['state'] == 'inactive'),
                   reverse=True)
    held = [torch.full((n // 4, ), SENTINEL, dtype=torch.float32, device=DEV) for n in sizes if n >= 4]
    torch.cuda.synchronize()
    del held


def twice_with_nan(losses, inputs):
    """two backward passes through one graph, all-NaN upstream gradients; -> the gradients of the second"""
    losses = [l for l in losses if l.requires_grad]
    nan = [torch.full_like(l, float('nan')) for l in losses]
    torch.autograd.grad(losses, inputs, nan, retain_graph=True)
    fill_free_blocks()
    return torch.autograd.grad(losses, inputs, nan)


def a2c():
    op, t, p = cases.a2c_case(1, 2000, 6, weight='tensor')
    d = cases.prepare(op, t, DEV)
    loss = b2.a2c_error(b2.a2c_data(d['logit'], d['action'], d['value'], d['adv'], d['return_'], d['weight']))
    return list(loss), [d['logit'], d['value']]


def a2cc():
    g = torch.Generator().manual_seed(2)
    mu, sigma = torch.randn(2000, 3, generator=g), torch.rand(2000, 3, generator=g) + 0.3
    d = {k: v.to(DEV).requires_grad_(True) for k, v in (('mu', mu), ('sigma', sigma),
                                                         ('value', torch.randn(2000, generator=g)))}
    action, adv, ret = (torch.randn(2000, 3, generator=g).to(DEV), torch.randn(2000, generator=g).to(DEV),
                        torch.randn(2000, generator=g).to(DEV))
    loss = b2.a2c_error_continuous(b2.a2c_data({'mu': d['mu'], 'sigma': d['sigma']}, action, d['value'], adv, ret, None))
    return list(loss), [d['mu'], d['sigma'], d['value']]


def ppoc(pretrained):
    op, t, p = cases.ppoc_case(3, 2000, 3, weight='tensor', pretrained=pretrained)
    d = cases.prepare(op, t, DEV)
    pre = {'mu': d['mu_pretrained'], 'sigma': d['sigma_pretrained']} if pretrained else None
    data = b2.ppo_data({'mu': d['mu_new'], 'sigma': d['sigma_new']}, {'mu': d['mu_old'], 'sigma': d['sigma_old']},
                       d['action'], d['value_new'], d['value_old'], d['adv'], d['return_'], d['weight'], pre)
    loss, _ = b2.ppo_error_continuous(data)
    return list(loss) if pretrained else list(loss)[:3], [d['mu_new'], d['sigma_new'], d['value_new']]


def vtrace():
    op, t, p = cases.vtrace_case(4, 40, 64, 6, weight='tensor')
    d = cases.prepare(op, t, DEV)
    loss = b2.vtrace_error_discrete_action(b2.vtrace_data(d['target_output'], d['behaviour_output'], d['action'],
                                                          d['value'], d['reward'], d['weight']), **p)
    return list(loss), [d['target_output'], d['value']]


def ppo_lm(dtype):
    d = po.make_inputs(2, 8, 1536, dtype, 'frac', True, 5, 1.0, False, device=DEV)
    new = d['logit_new'].detach().clone().requires_grad_(True)
    data = b2.ppo_policy_data(new, d['logit_old'], d['action'], d['adv'], d['weight'], d['logit_pretrained'])
    loss, _ = b2.ppo_policy_error(data, entropy_bonus=True)
    return list(loss), [new]


CALLS = {
    'a2c': a2c,
    'a2cc': a2cc,
    'ppoc': lambda: ppoc(False),
    'ppoc_pre': lambda: ppoc(True),
    'vtrace': vtrace,
    'ppo_lm_f32': lambda: ppo_lm(torch.float32),
    'ppo_lm_bf16': lambda: ppo_lm(torch.bfloat16),
}


@pytest.mark.parametrize('name', sorted(CALLS))
def test_repeated_backward_recomputes_with_nan_upstream_gradients(name):
    losses, inputs = CALLS[name]()
    for i, (x, g) in enumerate(zip(inputs, twice_with_nan(losses, inputs))):
        assert g.shape == x.shape
        g = g.float()
        if name == 'vtrace' and i == 1:  # value[T] only bootstraps the detached targets: its gradient is 0
            assert (g[-1] == 0).all()
            g = g[:-1]
        assert torch.isnan(g).all(), '%s: %d of %d entries are not NaN' % (name, int((~torch.isnan(g)).sum()), g.numel())


def test_vtrace_verify_launch_without_record_recomputes():
    """b200rl_vtrace_fwd_grad with verify = 1 and a null g_used, called directly: the launch writes the gradients for the
    actual upstream gradients, which match the CPU oracle"""
    T, B, N = 33, 64, 6
    mix = [0.3, 1.7, 0.2]
    op, t, p = cases.vtrace_case(6, T, B, N, weight='tensor', gamma=0.99, lambda_=0.95, rho_clip_ratio=0.9,
                                 c_clip_ratio=1.1, rho_pg_clip_ratio=1.3)
    tw = cases.prepare(op, t, 'cpu')
    sum(c * l for c, l in zip(mix, rl_oracle.vtrace_error_discrete_action(**tw, **p))).backward()
    d = {k: (v.to(DEV) if isinstance(v, torch.Tensor) else v) for k, v in t.items()}
    g = [torch.tensor(c, dtype=torch.float32, device=DEV) for c in mix]
    grad_logit = torch.full_like(d['target_output'], SENTINEL)
    grad_value = torch.full((T + 1, B), SENTINEL, dtype=torch.float32, device=DEV)
    ptr = ops.ptr
    with torch.cuda.device(DEV):
        ws = ops.workspace(d["target_output"].device)
        rc = ops.lib().b200rl_vtrace_fwd_grad(
            ptr(d['target_output']), ptr(d['behaviour_output']), ptr(d['action']), ptr(d['value']), ptr(d['reward']),
            ptr(d['weight']), T, B, N, p['gamma'], p['lambda_'], p['rho_clip_ratio'], p['c_clip_ratio'],
            p['rho_pg_clip_ratio'], None, 1, ptr(g[0]), ptr(g[1]), ptr(g[2]), None, None, None, ptr(grad_logit),
            ptr(grad_value), ptr(ws), ws.numel() * 4, ops.stream_ptr())
    assert rc == 0
    for got, want in ((grad_logit, tw['target_output'].grad), (grad_value, tw['value'].grad)):
        a, b = got.cpu().numpy(), want.numpy()
        assert np.allclose(a, b, rtol=1e-5, atol=1e-5 * np.abs(b).max())
