"""GPU suite (-m gpu): parity of the CUDA path (through the C ABI) against

1. the committed golden fixtures -- outputs of the unmodified reference (tests/golden/make_golden.py);
2. the CPU oracle on the same seeded inputs at the BASELINE.json sizes;
3. size-independent properties at full size, and the edge cases the reference's tests exercise.

Tolerances (north star): bit-exact for gae / lambda-returns / in-place masks (pure fp32 mul-add in reference order
and boolean-driven recurrences); |a-b| <= 1e-5 + 1e-5*|b| for everything that involves exp/log or a reduction.
"""
import numpy as np
import pytest
import torch

import di_engine_b200 as b2
from oracle import rl_oracle
from tests import cases, golden_io

pytestmark = pytest.mark.gpu
DEV = 'cuda'


def _run(op, tensors, params, device=DEV):
    return cases.run_api(b2.rl_utils, op, tensors, params, device=device)


@pytest.mark.parametrize('name', golden_io.names())
def test_matches_reference_golden(name):
    op, tensors, params, expected = golden_io.load(name)
    got = _run(op, tensors, params)
    if op in ('gae', 'retrace'):
        cases.compare(got, expected, exact=True)
    else:
        cases.compare(got, expected, rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize('name', golden_io.names())
def test_host_buffer_path_matches_golden(name):
    """CPU tensors in -> staged to the GPU -> results (and the in-place next_value mask) back on the host."""
    op, tensors, params, expected = golden_io.load(name)
    got = _run(op, tensors, params, device='cpu')
    cases.compare(got, expected, exact=(op in ('gae', 'retrace')))


BIG = {
    'gae_D': lambda: cases.gae_case(100, 128, 4096, p_done=0.01),
    'gae_D_none': lambda: cases.gae_case(105, 128, 4096, done=None, traj=None),
    'gae_long1d': lambda: cases.gae_case(106, 3200, 1, one_d=True, p_done=0.01),
    'gae_ragged': lambda: cases.gae_case(107, 131, 1001, p_done=0.05),
    'gae_T1024': lambda: cases.gae_case(108, 1024, 64, p_done=0.02),
    'ppo_D': lambda: cases.ppo_case(101, 128 * 4096, 6, clip_ratio=0.2),
    'ppo_D_w_dc': lambda: cases.ppo_case(109, 128 * 512 + 37, 6, weight='tensor', dual_clip=3.0),
    'ppo_N18_kl': lambda: cases.ppo_case(110, 10000, 18, pretrained=True, kl_type='k3', weight='tensor'),
    'ppo_N40': lambda: cases.ppo_case(111, 3000, 40, weight='tensor'),
    'ppo_N1000': lambda: cases.ppo_case(112, 257, 1000),
    'ppo_marl_big': lambda: cases.ppo_case(113, 2000, 9, A=5, weight='tensor'),
    'qntd_B': lambda: cases.qntd_case(102, 512, 6, 3, value_gamma='tensor', gamma=0.99, done='bern'),
    'qntd_big': lambda: cases.qntd_case(114, 100003, 18, 5, weight='tensor'),
    'qntdr_B': lambda: cases.qntd_case(115, 512, 6, 3, rescale=True, value_gamma='tensor', done='bern'),
    'dntd_C': lambda: cases.dntd_case(103, 512, 6, 51, 3, gamma=0.99, value_gamma='tensor'),
    'dntd_big': lambda: cases.dntd_case(116, 4099, 4, 51, 5, weight='tensor'),
    'tdl_hpc': lambda: cases.td_lambda_case(117, 1024, 64, weight='tensor'),
    'tdl_wide': lambda: cases.td_lambda_case(118, 64, 8192, gamma=0.99, lambda_=0.95),
    'upgo_big': lambda: cases.upgo_case(119, 64, 64, 64),
    'upgo_N200': lambda: cases.upgo_case(120, 16, 16, 200),
    'vtrace_E': lambda: cases.vtrace_case(104, 64, 8192, 6, gamma=0.99, lambda_=0.95),
    'vtrace_ragged': lambda: cases.vtrace_case(121, 130, 333, 7, weight='tensor', rho_clip_ratio=0.9),
    'vtrace_N100': lambda: cases.vtrace_case(122, 8, 16, 100),
    'happo_big': lambda: cases.happo_case(125, 128 * 512 + 37, 6, weight='tensor', dual_clip=3.0),
    'happo_N40': lambda: cases.happo_case(126, 3000, 40, weight='tensor'),
    'happo_marl_big': lambda: cases.happo_case(131, 2000, 9, A=5, weight='tensor'),
    'happoc_big': lambda: cases.happoc_case(129, 4099, 6, weight='tensor', dual_clip=2.0),
    'ppg_big': lambda: cases.ppg_case(130, 4099, 18, weight='tensor'),
    'acer_big': lambda: cases.acer_case(127, 64, 512, 6),
    'acer_N18': lambda: cases.acer_case(128, 33, 130, 18, c_clip_ratio=1.5, trust_region_value=0.05),
    'retrace_E': lambda: cases.retrace_case(123, 64, 8192, 6),
    'retrace_long': lambda: cases.retrace_case(124, 1003, 130, 18, gamma=0.997),
}


@pytest.mark.parametrize('name', sorted(BIG.keys()))
def test_matches_oracle_at_baseline_sizes(name):
    op, tensors, params = BIG[name]()
    want = cases.run_oracle(rl_oracle, op, tensors, params)
    got = _run(op, tensors, params)
    if op in ('gae', 'retrace'):
        cases.compare(got, want, exact=True)
    else:
        cases.compare(got, want, rtol=1e-5, atol=1e-5)


def test_lambda_returns_bit_exact_including_tensor_operands():
    g = torch.Generator().manual_seed(5)
    T, B = 97, 203
    v = torch.randn(T + 1, B, generator=g)
    r = torch.randn(T, B, generator=g)
    gam = torch.rand(T, B, generator=g)
    lam = torch.rand(T, B, generator=g)
    done = (torch.rand(T, B, generator=g) < 0.1).float()
    for args in ((0.99, 0.95, None), (gam, lam, None), (gam, 0.9, done), (1.0, lam > 0.5, done)):
        want = rl_oracle.generalized_lambda_returns(v, r, *args)
        dargs = [a.to(DEV) if isinstance(a, torch.Tensor) else a for a in args]
        got = b2.generalized_lambda_returns(v.to(DEV), r.to(DEV), *dargs).cpu()
        assert torch.equal(got, want)
    assert torch.equal(b2.upgo_returns(r.to(DEV), v.to(DEV)).cpu(), rl_oracle.upgo_returns(r, v))


def test_gae_unaligned_noncontiguous_and_inplace_semantics():
    op, t, p = cases.gae_case(7, 64, 260, p_done=0.1)
    want = cases.run_oracle(rl_oracle, op, t, p)
    # (a) views with an odd storage offset -> the scalar (non-float4) kernel path
    pad = {k: torch.cat([torch.zeros(1), v.reshape(-1)]).to(DEV)[1:].view(v.shape) for k, v in t.items()}
    adv = b2.gae(b2.gae_data(*pad.values()), **p)
    assert np.array_equal(adv.cpu().numpy(), want['out_adv'])
    assert np.array_equal(pad['next_value'].cpu().numpy(), want['out_next_value_after'])  # mutated in place
    # (b) non-contiguous (transposed storage) inputs: result identical, caller's next_value still masked
    nc = {k: v.t().contiguous().to(DEV).t() for k, v in t.items()}
    assert not nc['value'].is_contiguous()
    adv = b2.gae(b2.gae_data(*nc.values()), **p)
    assert np.array_equal(adv.cpu().numpy(), want['out_adv'])
    assert np.array_equal(nc['next_value'].cpu().numpy(), want['out_next_value_after'])


def test_gae_properties_at_full_size():
    T, B = 128, 4096
    g = torch.Generator().manual_seed(11)
    v, nv, r = (torch.randn(T, B, generator=g).to(DEV) for _ in range(3))
    # lambda = 0 -> adv is exactly the one-step TD residual (no recurrence)
    adv0 = b2.gae(b2.gae_data(v, nv.clone(), r, None, None), 0.99, 0.0)
    assert torch.equal(adv0, r + 0.99 * nv - v)
    # traj_flag = 1 everywhere cuts every trace: same result with any lambda
    ones = torch.ones(T, B, device=DEV)
    adv1 = b2.gae(b2.gae_data(v, nv.clone(), r, torch.zeros_like(ones), ones), 0.99, 0.95)
    assert torch.equal(adv1, adv0)
    # done = 1 everywhere: next_value is zeroed in place and adv = r - v (+ trace of the same)
    nv2 = nv.clone()
    adv2 = b2.gae(b2.gae_data(v, nv2, r, ones, ones), 0.99, 0.95)
    assert torch.count_nonzero(nv2) == 0 and torch.equal(adv2, r + 0.99 * nv2 - v)


def test_ppo_gradient_rows_sum_to_zero_at_full_size():
    """d loss / d logits of any function of a softmax sums to zero along the action axis."""
    op, t, p = cases.ppo_case(3, 128 * 4096, 6, weight='tensor')
    got = _run(op, t, p)
    gl = got['grad_logit_new'].astype(np.float64)
    assert np.abs(gl.sum(-1)).max() < 1e-9
    assert np.isfinite(gl).all() and np.abs(gl).max() > 0


def test_c51_projection_conserves_mass_at_full_size():
    op, t, p = cases.dntd_case(9, 512, 6, 51, 3, gamma=0.99)
    t = dict(t)
    t['dist'] = torch.full_like(t['dist'], 1.0 / 51)
    got = _run(op, t, p)
    assert np.allclose(got['out_td_error_per_sample'], np.log(51.0), atol=1e-5)


def test_c51_nonpositive_dist_raises_like_reference():
    op, t, p = cases.dntd_case(9, 8, 3, 51, 3)
    t = dict(t)
    t['dist'] = t['dist'].clone()
    t['dist'][2, t['act'][2], 7] = 0.0
    with pytest.raises(AssertionError):
        _run(op, t, p)


def test_repeated_calls_are_deterministic_and_workspace_is_reusable():
    op, t, p = cases.ppo_case(4, 70001, 6, weight='tensor')
    a = _run(op, t, p)
    for _ in range(3):
        b = _run(op, t, p)
        cases.compare(b, a, exact=True)


def test_criterion_variants_match_torch_modules():
    import torch.nn as nn
    op, t, p = cases.qntd_case(21, 257, 5, 3, weight='tensor')
    for crit in (nn.SmoothL1Loss(reduction='none', beta=0.7), nn.HuberLoss(reduction='none', delta=0.4),
                 nn.L1Loss(reduction='none')):
        tt = cases.prepare(op, t)
        want_l, want_p = rl_oracle.q_nstep_td_error(**tt, gamma=0.95, nstep=3, criterion=crit)
        want_l.backward()
        td = cases.prepare(op, t, DEV)
        data = b2.q_nstep_td_data(*[td[k] for k in ('q', 'next_n_q', 'action', 'next_n_action', 'reward', 'done',
                                                    'weight')])
        loss, per = b2.q_nstep_td_error(data, 0.95, nstep=3, criterion=crit)
        loss.backward()
        assert torch.allclose(loss.cpu(), want_l, rtol=1e-5, atol=1e-5)
        assert torch.allclose(per.cpu(), want_p, rtol=1e-5, atol=1e-5)
        assert torch.allclose(td['q'].grad.cpu(), tt['q'].grad, rtol=1e-5, atol=1e-6)


def test_cuda_graph_capture_of_the_learner_step():
    """gae -> ppo forward -> ppo backward recorded in one CUDA graph and replayed: same numbers as eager."""
    from di_engine_b200 import ops
    T, B, N = 128, 512, 6
    _, tg, pg = cases.gae_case(31, T, B, p_done=0.01)
    _, tp, pp = cases.ppo_case(32, T * B, N)
    tg = {k: v.to(DEV) for k, v in tg.items()}
    tp = {k: (v.to(DEV) if v is not None else None) for k, v in tp.items()}
    nv0 = tg['next_value'].clone()
    s = torch.cuda.Stream()
    outs = {}

    def step():
        tg['next_value'].copy_(nv0)
        adv = ops.gae_(tg['value'], tg['next_value'], tg['reward'], tg['done'], tg['traj_flag'], 0.99, 0.95, 1)
        ln = tp['logit_new'].detach().requires_grad_(True)
        vn = tp['value_new'].detach().requires_grad_(True)
        p, v, e, k, _ = ops.PPOFunction.apply(ln, vn, tp['logit_old'], tp['action'], tp['value_old'], adv.view(-1),
                                              tp['return_'], None, None, T * B, 1, N, 0.2, 1, 0.0, 1, 'ppo', None)
        (p + 0.5 * v - 0.01 * e).backward()
        outs.update(adv=adv, p=p, gl=ln.grad, gv=vn.grad)

    with torch.cuda.stream(s):
        for _ in range(2):
            step()
        eager = {k: v.clone() for k, v in outs.items()}
        s.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            step()
        for _ in range(3):
            graph.replay()
    s.synchronize()
    for k in eager:
        assert torch.equal(outs[k], eager[k]), k


def _ppo_with_mix(t, p, mix, device=DEV, retain=False):
    td = cases.prepare('ppo', t, device)
    data = b2.ppo_data(*[td[k] for k in ('logit_new', 'logit_old', 'action', 'value_new', 'value_old', 'adv',
                                           'return_', 'weight', 'logit_pretrained')])
    loss, info = b2.ppo_error(data, **p)
    total = sum(c * l for c, l in zip(mix, loss))
    total.backward(retain_graph=retain)
    return td, loss, total


def _ppo_oracle_with_mix(t, p, mix):
    tt = cases.prepare('ppo', t)
    out = rl_oracle.ppo_error(**tt, **p)
    sum(c * l for c, l in zip(mix, out[:4])).backward()
    return tt


def test_ppo_fused_backward_is_exact_for_any_upstream_gradient():
    """The forward pass pre-computes gradients for the loss mix it expects (learned from the previous backward);
    a different mix at backward time must still give the right gradients (device-side check + recompute)."""
    from di_engine_b200 import ops
    assert ops.PPO_FUSED_BACKWARD
    op, t, p = cases.ppo_case(77, 4099, 6, weight='tensor', pretrained=True, kl_type='k2')
    for mix in ([1.0, 0.5, -0.01, 0.3], [1.0, 0.5, -0.01, 0.3], [0.7, 2.0, 0.05, -1.5], [0.0, 1.0, 0.0, 0.0],
                [0.7, 2.0, 0.05, -1.5]):
        want = _ppo_oracle_with_mix(t, p, mix)
        td, _, _ = _ppo_with_mix(t, p, mix)
        for k in ('logit_new', 'value_new'):
            a, b = td[k].grad.cpu().numpy(), want[k].grad.numpy()
            assert np.allclose(a, b, rtol=1e-5, atol=1e-5 * np.abs(b).max()), (mix, k)
    # hint now equals the last mix: the expected path (no recompute) must give the same numbers
    td2, _, _ = _ppo_with_mix(t, p, [0.7, 2.0, 0.05, -1.5])
    ga, gb = td2['logit_new'].grad, td['logit_new'].grad
    assert torch.allclose(ga, gb, rtol=1e-5, atol=1e-5 * float(gb.abs().max()))


def test_ppo_repeated_backward_and_unfused_path_agree():
    from di_engine_b200 import ops
    op, t, p = cases.ppo_case(78, 1500, 5, weight='tensor')
    mix = [1.0, 0.5, -0.01, 0.0]
    td, loss, total = _ppo_with_mix(t, p, mix, retain=True)
    g1 = td['logit_new'].grad.clone()
    total.backward()  # second backward through the same graph accumulates the same gradient again
    assert torch.allclose(td['logit_new'].grad, 2 * g1, rtol=1e-6, atol=0)
    ops.PPO_FUSED_BACKWARD = False
    try:
        td3, _, _ = _ppo_with_mix(t, p, mix)
    finally:
        ops.PPO_FUSED_BACKWARD = True
    assert torch.allclose(td3['logit_new'].grad, g1, rtol=1e-6, atol=1e-12)
    assert torch.allclose(td3['value_new'].grad, td['value_new'].grad / 2, rtol=1e-6, atol=1e-12)
    with torch.no_grad():
        tn = cases.prepare('ppo', t, DEV)
        data = b2.ppo_data(*[tn[k].detach() if isinstance(tn[k], torch.Tensor) else tn[k] for k in (
            'logit_new', 'logit_old', 'action', 'value_new', 'value_old', 'adv', 'return_', 'weight',
            'logit_pretrained')])
        l2, _ = b2.ppo_error(data, **p)
    assert torch.allclose(l2.policy_loss, loss.policy_loss, rtol=1e-6)


def _fused_vs_oracle(T, B, N, seed, mix=(1.0, 0.5, -0.01, 0.0), done='float', traj='float', weight='none',
                     pretrained=False, grad=True, **pp):
    _, tg, pg = cases.gae_case(seed, T, B, done=done, traj=traj, p_done=0.03, gamma=0.99, lambda_=0.95)
    _, tp, _ = cases.ppo_case(seed + 1, T * B, N, weight=weight, pretrained=pretrained)
    # oracle: gae then ppo_error
    og = {k: (v.clone() if isinstance(v, torch.Tensor) else v) for k, v in tg.items()}
    adv_ref = rl_oracle.gae(og['value'], og['next_value'], og['reward'], og['done'], og['traj_flag'], **pg)
    tt = cases.prepare('ppo', tp)
    tt['adv'] = adv_ref.reshape(-1)
    out = rl_oracle.ppo_error(**tt, **pp)
    if grad:
        sum(c * l for c, l in zip(mix, out[:4])).backward()
    # product: one call
    dg = {k: (v.clone().to(DEV) if isinstance(v, torch.Tensor) else v) for k, v in tg.items()}
    td = cases.prepare('ppo', tp, DEV)
    if not grad:
        td = {k: (v.detach() if isinstance(v, torch.Tensor) else v) for k, v in td.items()}
    adv, loss, info = b2.gae_ppo_error(
        b2.gae_data(dg['value'], dg['next_value'], dg['reward'], dg['done'], dg['traj_flag']),
        b2.ppo_data(td['logit_new'], td['logit_old'], td['action'], td['value_new'], td['value_old'], None,
                    td['return_'], td['weight'], td['logit_pretrained']), pg['gamma'], pg['lambda_'], **pp)
    assert torch.equal(adv.cpu(), adv_ref), 'fused adv must be bit-identical to gae'
    assert torch.equal(dg['next_value'].cpu(), og['next_value']), 'in-place next_value mask'
    for got, want in zip(loss, out[:4]):
        assert torch.allclose(got.cpu(), want.detach(), rtol=1e-5, atol=1e-5)
    assert abs(info.approx_kl - out[4]) < 1e-5 and abs(info.clipfrac - out[5]) < 1e-5
    if grad:
        sum(c * l for c, l in zip(mix, loss)).backward()
        for k in ('logit_new', 'value_new'):
            a, b = td[k].grad.cpu().numpy(), tt[k].grad.numpy()
            assert np.allclose(a, b, rtol=1e-5, atol=1e-5 * np.abs(b).max()), k


@pytest.fixture(params=['row', 'col'])
def gae_ppo_impl(request):
    """run the one-launch step through each of its kernels: csrc/fused.cu (row tiles) and csrc/colws.cu (column tiles,
    warp-specialised; falls through to row tiles where its ring does not fit two CTAs per SM: N > 21, or N > 14 with
    logit_pretrained)"""
    from di_engine_b200 import ops
    old = ops.lib().b200rl_gae_ppo_set_impl({'row': 1, 'col': 2}[request.param])
    yield request.param
    ops.lib().b200rl_gae_ppo_set_impl(old)


# (64, 1024, 22): column tiles cannot take N = 22, so row tiles run it even at B >= 1024.  (128, 1056, N): T*B = 256 * 132 * 4
# selects 2 rows per thread in the row kernel, whose layout does not fit in shared memory at N = 28 (N = 20 with
# logit_pretrained): the row kernel must take 1 row per thread instead
@pytest.mark.parametrize('shape', [(128, 4096, 6), (128, 512, 6), (100, 36, 6), (300, 64, 4), (1, 8, 3), (33, 20, 11),
                                   (64, 260, 18), (7, 6, 6), (257, 48, 6), (32, 16, 2), (5, 4, 7), (129, 1028, 6),
                                   (64, 1024, 22), (128, 1056, 28), (128, 1056, 20, 'pretrained')])
def test_fused_gae_ppo_matches_oracle(shape, gae_ppo_impl):
    T, B, N = shape[:3]
    _fused_vs_oracle(T, B, N, seed=500 + T, pretrained='pretrained' in shape)


def test_fused_gae_ppo_auto_dispatch():
    _fused_vs_oracle(128, 2048, 6, 700)  # B >= 1024 -> column tiles
    _fused_vs_oracle(64, 512, 6, 701)    # -> row tiles
    _fused_vs_oracle(16, 64, 6, 702)     # tiny -> column tiles


def test_fused_gae_ppo_variants(gae_ppo_impl):
    _fused_vs_oracle(96, 128, 6, 600, weight='tensor', dual_clip=3.0)
    _fused_vs_oracle(96, 128, 5, 601, pretrained=True, kl_type='k3', mix=(1.0, 0.5, -0.01, 0.2))
    _fused_vs_oracle(96, 128, 15, 608, pretrained=True, kl_type='k2')  # too wide for column tiles -> row tiles
    _fused_vs_oracle(96, 128, 6, 602, done=None, traj=None, use_value_clip=False)
    _fused_vs_oracle(96, 128, 6, 603, mix=(0.3, 1.7, 0.2, 0.0))  # upstream gradients the kernel did not expect
    _fused_vs_oracle(96, 128, 6, 604, mix=(0.3, 1.7, 0.2, 0.0))  # ... and now expects
    _fused_vs_oracle(96, 128, 6, 605, grad=False)
    _fused_vs_oracle(40, 30, 6, 606)  # B % 4 != 0 -> falls back to the two separate operators
    _fused_vs_oracle(96, 128, 40, 607)  # N > 32 -> fallback


def test_fused_gae_ppo_repeatable_under_graph_capture(gae_ppo_impl):
    from di_engine_b200 import ops
    T, B, N = 128, 512, 6
    hb = __import__('bench').make_batch(3, T=T, B=B, N=N)
    d = {k: v.to(DEV) for k, v in hb.items()}
    nv0 = d['next_value'].clone()
    s = torch.cuda.Stream()
    res = {}

    def step():
        d['next_value'].copy_(nv0)
        ln = d['logit_new'].detach().requires_grad_(True)
        vn = d['value_new'].detach().requires_grad_(True)
        adv, p, v, e, k, _ = ops.GAEPPOFunction.apply(ln, vn, d['value'], d['next_value'], d['reward'], d['done'],
                                                      d['traj_flag'], d['logit_old'], d['action'], d['value_old'],
                                                      d['return_'], None, None, T, B, N, 0.99, 0.95, 0.2, 1, 0.0, 1)
        (p + 0.5 * v - 0.01 * e).backward()
        res.update(adv=adv, p=p, gl=ln.grad, gv=vn.grad)

    with torch.cuda.stream(s):
        for _ in range(3):
            step()
        eager = {k: v.clone() for k, v in res.items()}
        s.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            step()
        for _ in range(5):
            g.replay()
    s.synchronize()
    for k in eager:
        if k == 'p' and gae_ppo_impl == 'row':  # dynamic tile hand-out -> summation order may differ in the last bits
            assert torch.allclose(res[k], eager[k], rtol=1e-6, atol=1e-7), k
        else:
            assert torch.equal(res[k], eager[k]), k


def _vtrace_once(t, p, mix, device=DEV, retain=False, grad=True):
    td = cases.prepare('vtrace', t, device)
    if not grad:
        td = {k: (v.detach() if isinstance(v, torch.Tensor) else v) for k, v in td.items()}
    if device == 'cpu':
        loss = rl_oracle.vtrace_error_discrete_action(**td, **p)
    else:
        loss = b2.vtrace_error_discrete_action(b2.vtrace_data(td['target_output'], td['behaviour_output'], td['action'],
                                                              td['value'], td['reward'], td['weight']), **p)
    total = sum(c * l for c, l in zip(mix, loss))
    if grad:
        total.backward(retain_graph=retain)
    return td, loss, total


def _vtrace_close(td, tw, loss, lw):
    for got, want in zip(loss, lw):
        assert torch.allclose(got.detach().cpu(), want.detach(), rtol=1e-5, atol=1e-5)
    for k in ('target_output', 'value'):
        a, b = td[k].grad.cpu().numpy(), tw[k].grad.numpy()
        assert np.allclose(a, b, rtol=1e-5, atol=1e-5 * np.abs(b).max()), k


@pytest.fixture(params=['auto', 'resident'])
def vtrace_impl(request):
    """auto = streaming column tiles where they fit, else resident tiles; resident = resident tiles wherever they fit"""
    from di_engine_b200 import ops
    old = ops.lib().b200rl_vtrace_set_impl({'auto': 0, 'resident': 2}[request.param])
    yield request.param
    ops.lib().b200rl_vtrace_set_impl(old)


@pytest.mark.parametrize('shape', [(64, 8192, 6), (70, 48, 6), (16, 16, 2), (5, 4, 7), (33, 20, 11), (130, 1028, 6),
                                   (1, 8, 3), (40, 64, 12), (20, 4808, 3)])  # B > 4736: 32-column tiles (the last one 8 wide), ragged T
def test_vtrace_one_launch_kernel_matches_oracle(shape, vtrace_impl):
    """csrc/vtws.cu through the public operator: forward + gradients in one launch, device-verified backward"""
    T, B, N = shape
    from di_engine_b200 import ops
    op, t, p = cases.vtrace_case(900 + T, T, B, N, weight='tensor' if T % 2 else 'none', gamma=0.99, lambda_=0.95,
                                 rho_clip_ratio=0.9, c_clip_ratio=1.1, rho_pg_clip_ratio=1.3)
    L = ops.lib()
    d = cases.prepare('vtrace', t, DEV)
    assert L.b200rl_vtrace_fused_supported(ops.ptr(d['target_output']), ops.ptr(d['behaviour_output']),
                                           ops.ptr(d['action']), ops.ptr(d['value']), ops.ptr(d['reward']),
                                           ops.ptr(d['weight']), T, B, N, None, None) == 1
    for mix in ([1.0, 0.5, -0.01], [0.3, 1.7, 0.2], [0.3, 1.7, 0.2]):  # expected, unexpected, then expected again
        tw, lw, _ = _vtrace_once(t, p, mix, device='cpu')
        td, loss, _ = _vtrace_once(t, p, mix)
        _vtrace_close(td, tw, loss, lw)
    ops.vtrace_hint(torch.device(DEV)).copy_(torch.tensor([1.0, 0.5, -0.01]))


@pytest.mark.parametrize('shape', [(64, 64, 18), (32, 40, 32), (48, 16, 100), (300, 8, 6), (17, 8, 2)])
def test_vtrace_resident_tiles_take_wide_rows_and_odd_tiles(shape):
    """shapes the streaming kernel does not take (N > 14: no three-stage ring) or takes with one tile: resident tiles"""
    T, B, N = shape
    op, t, p = cases.vtrace_case(970 + T, T, B, N, weight='tensor' if T % 2 else 'none', gamma=0.99, lambda_=0.95,
                                 rho_clip_ratio=0.9, c_clip_ratio=1.1, rho_pg_clip_ratio=1.3)
    for mix in ([1.0, 0.5, -0.01], [0.3, 1.7, 0.2]):
        tw, lw, _ = _vtrace_once(t, p, mix, device='cpu')
        td, loss, _ = _vtrace_once(t, p, mix)
        _vtrace_close(td, tw, loss, lw)
    from di_engine_b200 import ops
    ops.vtrace_hint(torch.device(DEV)).copy_(torch.tensor([1.0, 0.5, -0.01]))


def test_vtrace_one_launch_repeated_backward_nograd_legacy_and_fallback():
    from di_engine_b200 import ops
    op, t, p = cases.vtrace_case(950, 48, 64, 6, weight='tensor')
    mix = [1.0, 0.5, -0.01]
    tw, lw, _ = _vtrace_once(t, p, mix, device='cpu')
    td, loss, total = _vtrace_once(t, p, mix, retain=True)
    g1 = td['target_output'].grad.clone()
    total.backward()  # second backward through the same graph accumulates the same gradient again
    assert torch.allclose(td['target_output'].grad, 2 * g1, rtol=1e-6, atol=0)
    with torch.no_grad():
        _, l2, _ = _vtrace_once(t, p, mix, grad=False)
    for got, want in zip(l2, lw):
        assert torch.allclose(got.cpu(), want.detach(), rtol=1e-5, atol=1e-5)
    ops.VTRACE_FUSED = False  # rows / scan / backward kernels of csrc/pg.cu
    try:
        td3, l3, _ = _vtrace_once(t, p, mix)
    finally:
        ops.VTRACE_FUSED = True
    _vtrace_close(td3, tw, l3, lw)
    assert torch.allclose(td3['target_output'].grad, g1, rtol=1e-5, atol=1e-9)
    # B % 4 != 0 -> not supported by the one-launch kernels -> pg.cu path; N = 18: resident tiles (no three-stage ring)
    for shape in ((20, 30, 6), (24, 64, 18)):
        op, t, p = cases.vtrace_case(951, *shape)
        tw, lw, _ = _vtrace_once(t, p, mix, device='cpu')
        td, loss, _ = _vtrace_once(t, p, mix)
        _vtrace_close(td, tw, loss, lw)


def test_vtrace_one_launch_under_graph_capture():
    op, t, p = cases.vtrace_case(960, 64, 512, 6)
    d = cases.prepare('vtrace', t, DEV)
    s = torch.cuda.Stream()
    res = {}

    def step():
        tgt = d['target_output'].detach().requires_grad_(True)
        val = d['value'].detach().requires_grad_(True)
        loss = b2.vtrace_error_discrete_action(b2.vtrace_data(tgt, d['behaviour_output'], d['action'], val, d['reward'],
                                                              None), **p)
        (loss.policy_loss + 0.5 * loss.value_loss - 0.01 * loss.entropy_loss).backward()
        res.update(p=loss.policy_loss, v=loss.value_loss, gl=tgt.grad, gv=val.grad)

    with torch.cuda.stream(s):
        for _ in range(3):
            step()
        eager = {k: v.clone() for k, v in res.items()}
        s.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            step()
        for _ in range(5):
            g.replay()
    s.synchronize()
    for k in eager:
        assert torch.equal(res[k], eager[k]), k


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='needs two GPUs')
def test_same_operators_on_two_devices_in_one_process():
    """The shared-memory opt-in of a kernel holds for one device only: run the one-launch gae -> ppo_error step
    (config D's N), ppo_error at N = 18 and the one-launch V-trace step (config E's N), whose kernels all need more than
    48 KB of dynamic shared memory, on cuda:0 and then cuda:1.  Every sum has a fixed order, so the results must be
    bit-identical across the devices."""
    _, tg, pg = cases.gae_case(41, 128, 4096, p_done=0.03)
    _, tp, pp = cases.ppo_case(42, 128 * 4096, 6)
    _, tq, pq = cases.ppo_case(43, 65536, 18)
    _, tv, pv = cases.vtrace_case(44, 64, 8192, 6)

    def run(dev):
        dg = {k: (v.clone().to(dev) if isinstance(v, torch.Tensor) else v) for k, v in tg.items()}
        td = cases.prepare('ppo', tp, dev)
        adv, loss, _ = b2.gae_ppo_error(
            b2.gae_data(dg['value'], dg['next_value'], dg['reward'], dg['done'], dg['traj_flag']),
            b2.ppo_data(td['logit_new'], td['logit_old'], td['action'], td['value_new'], td['value_old'], None,
                        td['return_'], td['weight'], td['logit_pretrained']), pg['gamma'], pg['lambda_'], **pp)
        sum(c * l for c, l in zip(cases.LOSS_MIX['ppo'], loss)).backward()
        tq_dev, loss_q, _ = _ppo_with_mix(tq, pq, cases.LOSS_MIX['ppo'], device=dev)
        tv_dev, loss_v, _ = _vtrace_once(tv, pv, (1.0, 0.5, -0.01), device=dev)
        out = {'adv': adv, 'gae_ppo_logit_grad': td['logit_new'].grad, 'gae_ppo_value_grad': td['value_new'].grad,
               'ppo_logit_grad': tq_dev['logit_new'].grad, 'ppo_value_grad': tq_dev['value_new'].grad,
               'vtrace_logit_grad': tv_dev['target_output'].grad, 'vtrace_value_grad': tv_dev['value'].grad}
        for name, ls in (('gae_ppo', loss), ('ppo', loss_q), ('vtrace', loss_v)):
            out.update({'%s_loss%d' % (name, i): l for i, l in enumerate(ls)})
        return {k: v.detach().cpu() for k, v in out.items()}

    first, second = run('cuda:0'), run('cuda:1')
    for k in first:
        assert torch.equal(first[k], second[k]), k


def test_c_abi_from_plain_c():
    """examples/c_abi_gae.c: gcc-compiled caller with cudaMalloc'd buffers and its own stream -- no torch in the process;
    gae must be bit-identical to the host recurrence, including the in-place next_value mask."""
    import subprocess
    import __graft_entry__ as ge
    exe = ge.build_c_example()
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, (r.returncode, r.stdout, r.stderr)
    assert '0 mismatching values' in r.stdout


def test_packed_batch_round_trip_and_use():
    """di_engine_b200.PackedBatch: one pinned buffer -> one H2D copy -> device views with the original shapes / dtypes, usable
    by the operators (alignment) and refreshed by the next upload."""
    hb = __import__('bench').make_batch(5, T=32, B=48, N=6)
    hb['weight'] = None
    pb = b2.PackedBatch(hb, DEV)
    assert pb.payload_bytes() == sum(v.numel() * v.element_size() for v in hb.values() if v is not None)
    d, ev = pb.upload()
    torch.cuda.current_stream().wait_event(ev)
    for k, v in hb.items():
        if v is None:
            assert d[k] is None
        else:
            assert d[k].dtype == v.dtype and d[k].shape == v.shape and d[k].data_ptr() % 256 == 0
            assert torch.equal(d[k].cpu(), v), k
    adv = b2.gae(b2.gae_data(d['value'], d['next_value'], d['reward'], d['done'], d['traj_flag']), 0.99, 0.95)
    ref = rl_oracle.gae(hb['value'], hb['next_value'].clone(), hb['reward'], hb['done'], hb['traj_flag'], 0.99, 0.95)
    assert torch.equal(adv.cpu(), ref)
    pb.host['reward'].mul_(2.0)  # the collector writes into the pinned views; the next upload carries the change
    d2, ev2 = pb.upload()
    torch.cuda.current_stream().wait_event(ev2)
    assert torch.equal(d2['reward'].cpu(), hb['reward'] * 2.0)


def test_p2p_allreduce_kernel_single_rank_degenerate():
    """world = 1: the mailbox exchange must reproduce the local values (mean over one rank), across many sequence
    numbers and under CUDA-graph replay.  (Two and more ranks: tests/test_p2p_gpu.py, tools/p2p_check.py under torchrun.)"""
    from di_engine_b200 import ops
    L = ops.lib()
    mailbox = torch.zeros(L.b200rl_p2p_mailbox_floats(1), device=DEV)
    ptrs = torch.tensor([mailbox.data_ptr()], dtype=torch.int64, device=DEV)
    seq = torch.zeros(1, dtype=torch.int32, device=DEV)
    out = torch.zeros(6, device=DEV)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        for it in range(5):
            src = torch.arange(8, device=DEV, dtype=torch.float32) + it
            rc = L.b200rl_p2p_allreduce_mean(src.data_ptr(), ptrs.data_ptr(), 0, 1, 6, seq.data_ptr(), out.data_ptr(),
                                             ops.stream_ptr())
            assert rc == 0
            s.synchronize()
            assert torch.equal(out, src[:6]) and int(seq.item()) == it + 1
        src = torch.full((8, ), 3.5, device=DEV)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            L.b200rl_p2p_allreduce_mean(src.data_ptr(), ptrs.data_ptr(), 0, 1, 6, seq.data_ptr(), out.data_ptr(),
                                        ops.stream_ptr())
        for _ in range(7):
            g.replay()
    s.synchronize()
    assert torch.equal(out, src[:6]) and int(seq.item()) == 12


# ----------------------------------------------------------------------------------------------------------------
# round 2: one-launch TD heads (forward also writes the unit-upstream gradient), attached td errors, sequence form,
# differentiable lambda returns
# ----------------------------------------------------------------------------------------------------------------
BIG_TD = {
    'bdq_big': lambda: cases.bdq_case(130, 4099, 6, 11, 3, weight='tensor', value_gamma='tensor'),
    'qseq_r2d2_size': lambda: cases.qseq_case(131, 75, 64, 6, 5),            # ding/policy/r2d2.py defaults on Atari
    'qseq_rescale_wide': lambda: cases.qseq_case(132, 40, 1031, 18, 3, rescale=True),
    'qseq_T1': lambda: cases.qseq_case(133, 1, 9, 3, 2, weight='none'),
    'd1td_big': lambda: cases.d1td_case(134, 2050, 6, 51),
}


@pytest.mark.parametrize('name', sorted(BIG_TD.keys()))
def test_td_siblings_match_oracle(name):
    op, tensors, params = BIG_TD[name]()
    want = cases.run_oracle(rl_oracle, op, tensors, params)
    got = _run(op, tensors, params)
    cases.compare(got, want, rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize('op_case', ['qntd', 'qntdr', 'dntd', 'bdq'])
def test_td_heads_exact_for_any_upstream_gradient(op_case):
    """The forward launch writes the gradient for a unit upstream gradient; any other upstream value (and gradients that
    arrive through td_error_per_sample) must be honoured by the backward launch; repeated backward accumulates."""
    if op_case == 'qntd':
        op, t, p = cases.qntd_case(140, 777, 6, 3, weight='tensor', value_gamma='tensor')
    elif op_case == 'qntdr':
        op, t, p = cases.qntd_case(141, 300, 5, 4, rescale=True, weight='tensor')
    elif op_case == 'bdq':
        op, t, p = cases.bdq_case(142, 130, 5, 4, 3, weight='tensor')
    else:
        op, t, p = cases.dntd_case(143, 260, 4, 51, 3, weight='tensor')
    gin = cases.GRAD_INPUTS[op][0]

    def run(api_kind, scale, use_td):
        dev = DEV if api_kind == 'b200' else 'cpu'
        tt = cases.prepare(op, t, dev)
        pp = dict(p)
        if api_kind == 'b200':
            if op == 'dntd':
                data = b2.dist_nstep_td_data(*[tt[k] for k in ('dist', 'next_n_dist', 'act', 'next_n_act', 'reward', 'done',
                                                                'weight')])
                loss, per = b2.dist_nstep_td_error(data, **pp)
            else:
                data = b2.q_nstep_td_data(*[tt[k] for k in ('q', 'next_n_q', 'action', 'next_n_action', 'reward', 'done',
                                                             'weight')])
                if 'value_gamma' in tt:
                    pp['value_gamma'] = tt['value_gamma']
                gamma = pp.pop('gamma')
                fn = {'qntd': b2.q_nstep_td_error, 'qntd_rescale': b2.q_nstep_td_error_with_rescale,
                      'bdq': b2.bdq_nstep_td_error}[op]
                loss, per = fn(data, gamma, **pp)
        else:
            fn = {'qntd': rl_oracle.q_nstep_td_error, 'qntd_rescale': rl_oracle.q_nstep_td_error_with_rescale,
                  'bdq': rl_oracle.bdq_nstep_td_error, 'dntd': rl_oracle.dist_nstep_td_error}[op]
            loss, per = fn(**tt, **pp)
        total = scale * loss
        if use_td and per.requires_grad:
            coef = torch.linspace(-1, 1, per.numel(), device=per.device).reshape(per.shape)
            total = total + (per * coef).sum()
        total.backward(retain_graph=True)
        g1 = tt[gin].grad.clone()
        total.backward()
        return g1, tt[gin].grad.clone()

    for scale, use_td in ((1.0, False), (2.5, False), (1.0, True), (0.0, True)):
        w1, w2 = run('oracle', scale, use_td)
        g1, g2 = run('b200', scale, use_td)
        for a, b in ((g1, w1), (g2, w2)):
            a, b = a.cpu().numpy(), b.numpy()
            assert np.allclose(a, b, rtol=1e-5, atol=1e-5 * max(np.abs(b).max(), 1e-30)), (op_case, scale, use_td)


QUANTILE_BIG = {
    'qrdqn_atari': lambda: cases.quantile_case(160, 'qrdqn', 64, 6, 200, 200, 3, weight='tensor'),   # num_quantiles 200
    'qrdqn_B600': lambda: cases.quantile_case(161, 'qrdqn', 600, 4, 32, 32, 1, value_gamma='tensor', tau='row'),
    'iqn_atari': lambda: cases.quantile_case(162, 'iqn', 64, 6, 32, 32, 3, weight='tensor', kappa=1.0),
    'iqn_ragged': lambda: cases.quantile_case(163, 'iqn', 37, 5, 150, 9, 5, value_gamma='scalar', kappa=0.3),
    'fqf_atari': lambda: cases.quantile_case(164, 'fqf', 64, 6, 32, 32, 3, weight='tensor'),
    'fqf_B1030': lambda: cases.quantile_case(165, 'fqf', 1030, 3, 8, 64, 2, value_gamma='tensor', kappa=2.0),
}


@pytest.mark.parametrize('name', sorted(QUANTILE_BIG.keys()))
def test_quantile_td_heads_match_oracle(name):
    op, tensors, params = QUANTILE_BIG[name]()
    want = cases.run_oracle(rl_oracle, op, tensors, params)
    got = _run(op, tensors, params)
    cases.compare(got, want, rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize('kind', ['qrdqn', 'iqn', 'fqf'])
def test_quantile_td_exact_for_any_upstream_gradient(kind):
    """unit-gradient buffer of the forward launch, any other upstream value, gradients through td_error_per_sample, and a
    repeated backward"""
    op, t, p = cases.quantile_case(170, kind, 70, 5, 16, 12, 3, weight='tensor', value_gamma='tensor')
    fields = cases.QUANTILE_FIELDS[op]

    def run(api_kind, scale, use_td):
        tt = cases.prepare(op, t, DEV if api_kind == 'b200' else 'cpu')
        if api_kind == 'b200':
            data = getattr(b2, kind + '_nstep_td_data')(*[tt[k] for k in fields])
            loss, per = getattr(b2, kind + '_nstep_td_error')(data, value_gamma=tt['value_gamma'], **p)
        else:
            loss, per = getattr(rl_oracle, kind + '_nstep_td_error')(*[tt[k] for k in fields], value_gamma=tt['value_gamma'], **p)
        total = scale * loss
        if use_td:
            total = total + (per * torch.linspace(-1, 1, per.numel(), device=per.device)).sum()
        total.backward(retain_graph=True)
        g1 = tt['q'].grad.clone()
        total.backward()
        return g1, tt['q'].grad.clone()

    for scale, use_td in ((1.0, False), (2.5, False), (1.0, True), (0.0, True)):
        w1, w2 = run('oracle', scale, use_td)
        g1, g2 = run('b200', scale, use_td)
        for a, b in ((g1, w1), (g2, w2)):
            a, b = a.cpu().numpy(), b.numpy()
            assert np.allclose(a, b, rtol=1e-5, atol=1e-5 * max(np.abs(b).max(), 1e-30)), (kind, scale, use_td)


@pytest.mark.parametrize('shape', [(33, 17, 6, None), (16, 16, 200, None), (12, 9, 5, 3)])
def test_upgo_head_exact_for_any_upstream_gradient(shape):
    """the forward launch writes the gradient for a unit upstream gradient in the same pass over the logits; any other upstream
    value and a repeated backward go through the recompute path"""
    T, B, N, N2 = shape
    op, t, p = cases.upgo_case(180 + N, T, B, N, N2=N2, mask=N2 is not None)
    for scale in (1.0, 2.5, 0.0):
        tw = cases.prepare(op, t)
        (scale * rl_oracle.upgo_loss(**tw)).backward()
        td = cases.prepare(op, t, DEV)
        loss = b2.upgo_loss(td['target_output'], td['rhos'], td['action'], td['rewards'], td['bootstrap_values'], td['mask'])
        total = scale * loss
        total.backward(retain_graph=True)
        g1 = td['target_output'].grad.clone()
        total.backward()
        b = tw['target_output'].grad.numpy()
        for a, f in ((g1, 1.0), (td['target_output'].grad, 2.0)):
            assert np.allclose(a.cpu().numpy(), f * b, rtol=1e-5, atol=1e-5 * max(np.abs(b).max(), 1e-30)), (shape, scale, f)


def test_lambda_returns_backward_matches_autograd_of_the_recurrence():
    """Gradients w.r.t. values, rewards and tensor gammas / lambdas against autograd of an out-of-place restatement
    (the reference's in-place loop supports the first two; MBSAC needs them, mbpolicy/mbsac.py:137,153); UPGO mode too."""
    g = torch.Generator().manual_seed(150)
    for T, B in ((17, 33), (130, 260), (1, 5), (64, 1)):
        v = torch.randn(T + 1, B, generator=g)
        r = torch.randn(T, B, generator=g)
        gam = torch.rand(T, B, generator=g)
        lam = torch.rand(T, B, generator=g)
        done = (torch.rand(T, B, generator=g) < 0.1).float()
        w = torch.randn(T, B, generator=g)
        for use_t, dn in ((True, done), (False, None), (True, None)):
            leaves_c = [x.clone().requires_grad_(True) for x in (v, r, gam, lam)]
            leaves_d = [x.clone().to(DEV).requires_grad_(True) for x in (v, r, gam, lam)]
            if use_t:
                want = rl_oracle.lambda_returns_functional(leaves_c[0], leaves_c[1], leaves_c[2], leaves_c[3], dn)
                got = b2.generalized_lambda_returns(leaves_d[0], leaves_d[1], leaves_d[2], leaves_d[3],
                                                    None if dn is None else dn.to(DEV))
            else:
                want = rl_oracle.lambda_returns_functional(leaves_c[0], leaves_c[1], 0.97, 0.9, dn)
                got = b2.generalized_lambda_returns(leaves_d[0], leaves_d[1], 0.97, 0.9, dn)
            assert torch.equal(got.detach().cpu(), rl_oracle.generalized_lambda_returns(
                v, r, gam if use_t else 0.97, lam if use_t else 0.9, dn)), 'forward stays bit-exact'
            (want * w).sum().backward()
            (got * w.to(DEV)).sum().backward()
            for a, b in zip(leaves_d[:4 if use_t else 2], leaves_c):
                a = a.grad.cpu().numpy()
                b = b.grad.numpy() if b.grad is not None else np.zeros_like(a)  # T = 1: lambda never enters the result
                assert np.allclose(a, b, rtol=1e-5, atol=1e-5 * max(np.abs(b).max(), 1e-30)), (T, B, use_t)
        # upgo_returns: gradient to rewards and bootstrap values, none through the comparison
        vc, rc = v.clone().requires_grad_(True), r.clone().requires_grad_(True)
        lambdas = (rc + vc[1:]) >= vc[:-1]
        lambdas = torch.cat([lambdas[1:], torch.ones_like(lambdas[-1:])], dim=0)
        want = rl_oracle.lambda_returns_functional(vc, rc, 1.0, lambdas.float())
        vd, rd = v.clone().to(DEV).requires_grad_(True), r.clone().to(DEV).requires_grad_(True)
        got = b2.upgo_returns(rd, vd)
        assert torch.equal(got.detach().cpu(), rl_oracle.upgo_returns(r, v))
        (want * w).sum().backward()
        (got * w.to(DEV)).sum().backward()
        for a, b in ((vd, vc), (rd, rc)):
            a, b = a.grad.cpu().numpy(), b.grad.numpy()
            assert np.allclose(a, b, rtol=1e-5, atol=1e-5 * max(np.abs(b).max(), 1e-30)), (T, B, 'upgo')


def test_tb_cross_entropy_matches_torch():
    g = torch.Generator().manual_seed(151)
    for shape, masked in (((9, 7, 6), False), ((5, 4, 3, 11), True), ((3, 2, 2, 130), False)):
        logit = torch.randn(*shape, generator=g)
        label = torch.randint(0, shape[-1], shape[:-1], generator=g)
        mask = (torch.rand(*shape[:-1], generator=g) > 0.3).float() if masked else None
        lc = logit.clone().requires_grad_(True)
        want = rl_oracle.tb_cross_entropy(lc, label, mask)
        ld = logit.clone().to(DEV).requires_grad_(True)
        got = b2.tb_cross_entropy(ld, label.to(DEV), None if mask is None else mask.to(DEV))
        assert got.shape == want.shape
        assert torch.allclose(got.detach().cpu(), want.detach(), rtol=1e-5, atol=1e-5)
        w = torch.randn(*want.shape, generator=g)
        (want * w).sum().backward()
        (got * w.to(DEV)).sum().backward()
        assert torch.allclose(ld.grad.cpu(), lc.grad, rtol=1e-5, atol=1e-6)


def test_ppo_fallback_grid_is_bounded_for_large_batches():
    """N > 64 takes the warp-per-row kernel: its grid (and workspace need) used to grow with S (ADVICE r1); 300k rows x 70."""
    op, t, p = cases.ppo_case(152, 300000, 70)
    t = {k: (v if v is None else v) for k, v in t.items()}
    want = cases.run_oracle(rl_oracle, op, t, p)
    got = _run(op, t, p)
    cases.compare(got, want, rtol=1e-5, atol=1e-5)


# ----------------------------------------------------------------------------------------------------------------
# SURVEY section 8f rank 1: the batch-level pieces around gae / ppo_error in PPOPolicy._forward_learn (policy/ppo.py:274-306)
# ----------------------------------------------------------------------------------------------------------------
def _learner_sequence(seed, T, n_env=8, p_done=0.003, flags=True):
    """ONE sequence of n_sample steps as the serial collector delivers it: n_env trajectories back to back, traj_flag = 1 at the
    end of each (and at every done), ding/policy/ppo.py:279-281"""
    g = torch.Generator().manual_seed(seed)
    value, next_value, reward = (torch.randn(T, generator=g) for _ in range(3))
    done = (torch.rand(T, generator=g) < p_done).float()
    traj = done.clone()
    if flags:
        seg = max(1, T // n_env)
        traj[seg - 1::seg] = 1.0
    traj[-1] = 1.0
    return value, next_value, reward, done, traj


@pytest.mark.parametrize('case', ['n_sample_3200', 'with_value_norm', 'no_flags_one_segment', 'every_step_an_end', 'T1',
                                  'T24576', 'batched_128x4096', 'batched_value_norm_ragged',
                                  'batched_small_value_norm'])
def test_gae_returns_matches_policy_lines(case):
    std = None
    if case == 'n_sample_3200':
        data = _learner_sequence(200, 3200)
    elif case == 'with_value_norm':
        data, std = _learner_sequence(201, 3200, p_done=0.01), 2.236068
    elif case == 'no_flags_one_segment':
        data = _learner_sequence(202, 5000, p_done=0.0, flags=False)
    elif case == 'every_step_an_end':
        v, nv, r, d, tf = _learner_sequence(203, 2000)
        data = (v, nv, r, d, torch.ones_like(tf))
    elif case == 'T1':
        data = _learner_sequence(204, 1)
    elif case == 'T24576':
        data = _learner_sequence(205, 24576, n_env=64)
    elif case == 'batched_128x4096':
        _, t, _ = cases.gae_case(206, 128, 4096, p_done=0.01)
        data = tuple(t.values())
    elif case == 'batched_value_norm_ragged':
        _, t, _ = cases.gae_case(207, 67, 1001, p_done=0.05)
        data, std = tuple(t.values()), 0.37
    else:
        _, t, _ = cases.gae_case(208, 33, 36, p_done=0.03)
        data, std = tuple(t.values()), 1.5
    want = rl_oracle.ppo_policy_gae_returns(*[x.clone() for x in data], 0.99, 0.95, std)
    dev = [x.clone().to(DEV) for x in data]
    got = b2.gae_returns(b2.gae_data(*dev), 0.99, 0.95, value_norm_std=std)
    for name, a, b in zip(got._fields[:4], got[:4], want[:4]):
        assert torch.equal(a.cpu(), b), name  # pure fp32 mul / add / div in the reference's order: bit-exact
    for x, y in zip(dev, data):
        assert torch.equal(x.cpu(), y), 'inputs must not be modified'
    st = got.return_stats.cpu().numpy().astype(np.float64)
    assert np.allclose(st, np.array(want[4]), rtol=2e-6, atol=1e-6), (st, want[4])
    if want[0].numel() > 1:  # adv.mean(), adv.std() + 1e-8 out of the same pass (policy/ppo.py:304-306 for a one-minibatch batch)
        a64 = want[0].double()
        ast = got.adv_stats.cpu().numpy().astype(np.float64)
        assert np.allclose(ast, [a64.mean().item(), a64.std().item() + 1e-8], rtol=2e-6, atol=1e-6), ast
    # plain gae on one sequence takes the same segment-parallel kernel: identical advantage, in-place mask as the reference
    dev2 = [x.clone().to(DEV) for x in data]
    if std is None:
        adv = b2.gae(b2.gae_data(*dev2), 0.99, 0.95)
        ref_in = [x.clone() for x in data]
        assert torch.equal(adv.cpu(), rl_oracle.gae(*ref_in, 0.99, 0.95))
        assert torch.equal(dev2[1].cpu(), ref_in[1]), 'next_value masked in place'


@pytest.mark.parametrize('S,N', [(320, 6), (64, 6), (524288, 6), (1000, 40)])
def test_ppo_error_adv_norm_matches_policy_lines(S, N):
    op, t, p = cases.ppo_case(210 + N, S, N, weight='tensor', clip_ratio=0.2)
    t = dict(t)
    t['adv'] = t['adv'] * 3.0 + 0.7  # far from normalised
    tt = cases.prepare('ppo', t)
    tt['adv'] = rl_oracle.normalize_advantage(tt['adv'])
    out = rl_oracle.ppo_error(**tt, **p)
    mix = cases.LOSS_MIX['ppo']
    sum(c * l for c, l in zip(mix, out[:4])).backward()
    td = cases.prepare('ppo', t, DEV)
    data = b2.ppo_data(*[td[k] for k in ('logit_new', 'logit_old', 'action', 'value_new', 'value_old', 'adv', 'return_',
                                           'weight', 'logit_pretrained')])
    loss, info = b2.ppo_error_adv_norm(data, **p)
    for got, want in zip(loss, out[:4]):
        assert torch.allclose(got.cpu(), want.detach(), rtol=1e-5, atol=1e-5)
    assert abs(info.approx_kl - out[4]) < 1e-5 and abs(info.clipfrac - out[5]) < 2e-5
    sum(c * l for c, l in zip(mix, loss)).backward()
    for k in ('logit_new', 'value_new'):
        a, b = td[k].grad.cpu().numpy(), tt[k].grad.numpy()
        assert np.allclose(a, b, rtol=1e-5, atol=1e-5 * np.abs(b).max()), k
    na = b2.normalize_advantage(td['adv'])
    assert torch.allclose(na.cpu(), tt['adv'], rtol=1e-6, atol=1e-6)
    # statistics handed in (e.g. gae_returns(...).adv_stats): same losses, no statistics launch
    stats = torch.stack([td['adv'].mean(), td['adv'].std() + 1e-8])
    loss2, _ = b2.ppo_error_adv_norm(data, adv_stats=stats, **p)
    for got, want in zip(loss2, out[:4]):
        assert torch.allclose(got.cpu(), want.detach(), rtol=1e-5, atol=1e-5)


def test_impala_reshape_data_then_vtrace_matches_policy_lines():
    """IMPALAPolicy._reshape_data masking (policy/impala.py:316-322) in front of vtrace_error_discrete_action: values, losses
    and the gradient that flows back THROUGH the mask to the critic output."""
    g = torch.Generator().manual_seed(220)
    for T, B, N in ((64, 8192, 6), (33, 257, 7)):
        tgt = torch.randn(T, B, N, generator=g)
        beh = tgt + 0.5 * torch.randn(T, B, N, generator=g)
        act = torch.randint(0, N, (T, B), generator=g)
        val = torch.randn(T + 1, B, generator=g)
        rew = torch.rand(T, B, generator=g)
        done = (torch.rand(T, B, generator=g) < 0.05).float()
        vc, tc = val.clone().requires_grad_(True), tgt.clone().requires_grad_(True)
        v2, r2, w2 = rl_oracle.impala_reshape_data(vc, rew, done)
        want = rl_oracle.vtrace_error_discrete_action(tc, beh, act, v2, r2, w2, gamma=0.99, lambda_=0.95)
        (want[0] + 0.5 * want[1] - 0.01 * want[2]).backward()
        vd, td = val.clone().to(DEV).requires_grad_(True), tgt.clone().to(DEV).requires_grad_(True)
        v3, r3, w3 = b2.impala_reshape_data(vd, rew.to(DEV), done.to(DEV))
        assert torch.equal(v3.detach().cpu(), v2.detach()) and torch.equal(r3.cpu(), r2) and torch.equal(w3.cpu(), w2)
        got = b2.vtrace_error_discrete_action(b2.vtrace_data(td, beh.to(DEV), act.to(DEV), v3, r3, w3), 0.99, 0.95)
        for a, b in zip(got, want):
            assert torch.allclose(a.cpu(), b.detach(), rtol=1e-5, atol=1e-5)
        (got[0] + 0.5 * got[1] - 0.01 * got[2]).backward()
        for a, b in ((vd, vc), (td, tc)):
            a, b = a.grad.cpu().numpy(), b.grad.numpy()
            assert np.allclose(a, b, rtol=1e-5, atol=1e-5 * np.abs(b).max())
