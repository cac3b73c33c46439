"""The PPO tile kernel (csrc/ppo.cu: ppo_tile_kernel, one CTA per SM over contiguous row spans) through the C ABI:
FWD, FWD_GRAD and the BWD recompute against a float64 torch reference at the geometry's edges (one row, one stage, a row
either side of a stage and of a span boundary, config P's 524 288 rows and a ragged tail), N in {1, 2, 6, 18, 32}, with
and without logit_pretrained, weight, HAPPO's factor and the advantage statistics; config P's three calls captured in
one CUDA graph against the same calls made eagerly; and the host geometry picker (no GPU needed)."""
import ctypes

import pytest
import torch

from di_engine_b200 import _lib, ops

CLIP = 0.2
STAGE_ROWS = 256


def _geometry(S, N, pre=False, w=False, verify=False, sms=132):
    g = (ctypes.c_longlong * 3)()
    assert _lib.load().b200rl_ppo_tile_geometry(S, N, int(pre), int(w), int(verify), sms, g) == 0
    return {'grid': g[0], 'stages': g[1], 'smem': g[2]}


def test_geometry_one_cta_per_sm_and_a_ring_from_the_smem_budget():
    for N in range(1, 33):
        for pre in (False, True):
            for w in (False, True):
                g = _geometry(524288, N, pre, w)
                assert g['grid'] == 132 and 1 <= g['stages'] <= 8 and g['smem'] <= 227 * 1024 - 1024, (N, pre, w, g)
    assert _geometry(524288, 6)['stages'] == 8  # config P: 18 KB stages
    assert _geometry(524288, 32)['stages'] >= 2
    # small batches: fewer CTAs, a ring no deeper than a CTA's tiles
    assert _geometry(64, 6)['grid'] == 1 and _geometry(64, 6)['stages'] == 1
    assert _geometry(320, 6)['grid'] == 2 and _geometry(320, 6)['stages'] == 1
    assert _geometry(3 * 132 * 256, 6)['stages'] == 3
    # the verification launch behind a fused forward: one stage, never more shared memory than the forward
    for N in (1, 6, 18, 32):
        v, f = _geometry(524288, N, verify=True), _geometry(524288, N)
        assert v['stages'] == 1 and v['grid'] == f['grid'] and v['smem'] < f['smem']
        assert v['smem'] <= 34 * 1024 or N > 6
    assert _geometry(524288, 6, verify=True)['smem'] <= 20 * 1024
    assert _lib.load().b200rl_ppo_tile_geometry(0, 6, 0, 0, 0, 132, (ctypes.c_longlong * 3)()) != 0


def _inputs(S, N, seed, pre, w, fac, stats, dev='cuda'):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g)  # noqa: E731
    t = {'logit_new': r(S, N), 'action': torch.randint(0, N, (S, ), generator=g), 'value_new': r(S), 'adv': r(S),
         'return_': 2 * r(S)}
    t['logit_old'] = t['logit_new'] + 0.1 * torch.rand(S, N, generator=g)
    t['value_old'] = t['value_new'] + 0.1 * torch.rand(S, generator=g)
    t['logit_pre'] = t['logit_new'] + 0.3 * r(S, N) if pre else None
    t['weight'] = torch.rand(S, generator=g) if w else None
    t['factor'] = 0.5 + torch.rand(S, generator=g) if fac else None
    t['adv_stats'] = torch.tensor([0.1, 1.3]) if stats else None
    return {k: (v.to(dev) if v is not None else None) for k, v in t.items()}


def _reference(t, mix):
    """float64: the six losses and d(sum mix_k * loss_k)/d(logit_new, value_new)"""
    d = {k: (v.double() if v is not None and v.is_floating_point() else v) for k, v in t.items()}
    ln = d['logit_new'].clone().requires_grad_(True)
    vn = d['value_new'].clone().requires_grad_(True)
    act = d['action'].unsqueeze(1)
    lp_n = torch.log_softmax(ln, 1)
    lp_o = torch.log_softmax(d['logit_old'], 1)
    lpa_n, lpa_o = lp_n.gather(1, act).squeeze(1), lp_o.gather(1, act).squeeze(1)
    adv = d['adv']
    if d['adv_stats'] is not None:
        adv = (adv - d['adv_stats'][0]) / d['adv_stats'][1]
    ratio = torch.exp(lpa_n - lpa_o)
    sel = torch.min(ratio * adv, ratio.clamp(1 - CLIP, 1 + CLIP) * adv)
    if d['factor'] is not None:
        sel = sel * d['factor']
    w = d['weight'] if d['weight'] is not None else torch.ones_like(adv)
    vc = d['value_old'] + (vn - d['value_old']).clamp(-CLIP, CLIP)
    vt = torch.max((d['return_'] - vn) ** 2, (d['return_'] - vc) ** 2)
    ent = -(lp_n.exp() * lp_n).sum(1)
    kl = (lpa_n - torch.log_softmax(d['logit_pre'], 1).gather(1, act).squeeze(1)).mean() if d['logit_pre'] is not None \
        else torch.zeros((), dtype=torch.float64, device=ln.device)
    losses = [-(sel * w).mean(), 0.5 * (vt * w).mean(), (ent * w).mean(), kl]
    sum(m * l for m, l in zip(mix, losses)).backward()
    info = [(lpa_o - lpa_n).mean(), ((ratio > 1 + CLIP) | (ratio < 1 - CLIP)).double().mean()]
    return torch.stack([x.detach() for x in losses + info]), ln.grad, vn.grad


def _args(t, S, N):
    p = ops.ptr
    return (p(t['logit_new']), p(t['logit_old']), p(t['logit_pre']), p(t['action']), p(t['value_new']), p(t['value_old']),
            p(t['adv']), p(t['return_']), p(t['weight']), S, 1, N, CLIP, 1, 0.0, 1, p(t['adv_stats']), p(t['factor']))


def _close(a, b, what):
    b = b.float()
    scale = float(b.abs().max()) if b.numel() else 1.0
    assert torch.allclose(a, b, rtol=1e-5, atol=1e-5 * max(scale, 1e-30)), (what, float((a - b).abs().max()), scale)


def _run_all(S, N, pre, w, fac, stats, seed):
    lib = _lib.load()
    t = _inputs(S, N, seed, pre, w, fac, stats)
    dev = t['logit_new'].device
    mix = [1.0, 0.5, -0.01, 0.3 if pre else 0.0]
    want_l, want_g, want_v = _reference(t, mix)
    ws = ops.workspace(dev)
    args = _args(t, S, N)
    # FWD
    out = torch.zeros(8, device=dev)
    assert lib.b200rl_ppo_fwd(*args, ops.ptr(out), ops.ptr(ws), ws.numel() * 4, ops.stream_ptr()) == 0
    torch.cuda.synchronize()
    for k in range(6):
        if k == 3 and not pre:
            continue
        assert abs(float(out[k]) - float(want_l[k])) <= 1e-5 + 1e-5 * abs(float(want_l[k])), (k, float(out[k]), float(want_l[k]))
    # FWD_GRAD for the expected mix, then the check (nothing recomputed) and a recompute under another mix
    expected = torch.tensor(mix, device=dev)
    used, hint = torch.zeros(4, device=dev), torch.zeros(4, device=dev)
    out2 = torch.zeros(8, device=dev)
    gl, gv = torch.full((S, N), float('nan'), device=dev), torch.full((S, ), float('nan'), device=dev)
    assert lib.b200rl_ppo_fwd_grad(*args, ops.ptr(expected), ops.ptr(used), ops.ptr(out2), ops.ptr(gl), ops.ptr(gv),
                                   ops.ptr(ws), ws.numel() * 4, ops.stream_ptr()) == 0
    torch.cuda.synchronize()
    assert torch.equal(out2[:6], out[:6])
    _close(gl, want_g, 'grad_logit fwd_grad')
    _close(gv, want_v, 'grad_value fwd_grad')
    g = [torch.tensor(m, device=dev) for m in mix]
    assert lib.b200rl_ppo_bwd(*args, *[ops.ptr(x) for x in g], ops.ptr(used), ops.ptr(hint), ops.ptr(gl), ops.ptr(gv),
                              ops.stream_ptr()) == 0
    torch.cuda.synchronize()
    _close(gl, want_g, 'grad_logit after check')
    mix2 = [0.7, 2.0, 0.05, -1.5 if pre else 0.0]
    _, want_g2, want_v2 = _reference(t, mix2)
    g2 = [torch.tensor(m, device=dev) for m in mix2]
    for rec in (used, None):  # the verify launch's one-stage recompute, and the plain backward
        gl.fill_(float('nan'))
        gv.fill_(float('nan'))
        assert lib.b200rl_ppo_bwd(*args, *[ops.ptr(x) for x in g2], ops.ptr(rec), ops.ptr(hint), ops.ptr(gl), ops.ptr(gv),
                                  ops.stream_ptr()) == 0
        torch.cuda.synchronize()
        _close(gl, want_g2, 'grad_logit recompute')
        _close(gv, want_v2, 'grad_value recompute')


def _span_edges():
    sms = torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132
    return [sms * STAGE_ROWS - 1, sms * STAGE_ROWS, sms * STAGE_ROWS + 1, 2 * sms * STAGE_ROWS + 1]


OPTS = [(False, False, False, False), (True, True, False, True), (False, True, True, False), (True, False, True, True)]


@pytest.mark.gpu
@pytest.mark.parametrize('S', [1, 127, 128, 129, 255, 256, 257, 4097, 50000, 70001] + _span_edges() +
                         [524288, 524288 + 37])
def test_rows_at_geometry_edges(S):
    for i, (pre, w, fac, stats) in enumerate(OPTS if S < 100000 else OPTS[:2]):
        _run_all(S, 6, pre, w, fac, stats, seed=S + i)


@pytest.mark.gpu
@pytest.mark.parametrize('N', [1, 2, 6, 18, 32])
@pytest.mark.parametrize('S', [300, 70001])
def test_row_widths_and_operands(N, S):
    for i, (pre, w, fac, stats) in enumerate(OPTS):
        _run_all(S, N, pre, w, fac, stats, seed=10 * N + S + i)


@pytest.mark.gpu
@pytest.mark.parametrize('N', [18, 32])
def test_wide_rows_at_config_p_size(N):
    _run_all(524288 + 37, N, True, True, False, True, seed=N)


# ---- config P's three calls under graph capture -----------------------------------------------------------------------
def _p_sets(n, T=128, B=512):
    import bench
    wl = bench.WorkloadP(B=B, T=T, N=6)
    return [wl.device_step(wl.make_batch(100 + i), 'cuda') for i in range(n)]


def _outputs(sets):
    return [{k: v.clone() for k, v in s.outputs().items()} for s in sets]


@pytest.mark.gpu
@pytest.mark.parametrize('order', ['rotated', 'same_twice', 'torch_op_between', 'reads_previous_outputs'])
def test_config_p_graph_matches_eager(order):
    sets = _p_sets(4)
    for s in sets[1:]:
        s.ws = torch.zeros_like(sets[0].ws)
    if order == 'reads_previous_outputs':  # step k + 1 takes step k's logit gradient as its logit_old
        for a, b in zip(sets[:-1], sets[1:]):
            b.b['logit_old'] = a.grad_logit
    seq = {'rotated': [0, 1, 2, 3, 0, 1, 2, 3], 'same_twice': [0, 0, 1, 1, 2, 2, 3, 3],
           'torch_op_between': [0, 1, 2, 3, 0, 1, 2, 3], 'reads_previous_outputs': [0, 1, 2, 3, 0, 1, 2, 3]}[order]
    init = [{k: v.clone() for k, v in s.b.items()} for s in sets]

    def restore():
        for s, b in zip(sets, init):
            for k, v in b.items():
                s.b[k].copy_(v)

    def run():
        res = []
        for i, k in enumerate(seq):
            if order == 'torch_op_between':
                nxt = sets[seq[(i + 1) % len(seq)]]
                nxt.b['logit_new'].mul_(0.75).add_(0.01 * i)
            sets[k]()
            res.append({n: v.clone() for n, v in sets[k].outputs().items()})
        return res

    main = torch.cuda.Stream()
    with torch.cuda.stream(main):
        restore()
        eager = run()
        main.synchronize()
        restore()
        main.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=main):
            captured = run()
        restore()
        main.synchronize()
        g.replay()
        main.synchronize()
    for i, (a, b) in enumerate(zip(eager, captured)):
        for k in a:
            assert torch.equal(a[k], b[k]), (order, i, k)
