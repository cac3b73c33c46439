"""The PPO-family and V-trace kernels against a float64 reference, on batches that run every branch of the policy math.

The seeded parity cases draw ``logit_old`` within 0.1 of ``logit_new``: no ratio is clipped, the dual-clip floor and the
clipped value branch never fire, and every logit is finite.  The generator below draws each row from one of four regimes
(on-policy, in band, clipped, far off-policy), masks illegal actions with ``-1e8`` or ``-inf`` as DI-engine's models do,
saturates some rows and shifts every row by its own constant.

Reference: ``cases.run_oracle`` on float64 copies of the same inputs (every fp32 value is exact in double).  The fp32 oracle
on the fp32 inputs is the yardstick: for every output X,

    max|X_gpu - X_64| <= K * max(max|X_32 - X_64|, 2^-24 * scale_X)

with ``scale_X = max|X_64|`` for a gradient and the fp64 mean of the per-sample |term| for a loss.  Rows on a branch
boundary of the fp64 reference (ratio at fp32(1 +- clip) or at the dual-clip floor, |dv| at the value clip, the two
value errors equal) may take the other branch in fp32: their gradients are left out of the elementwise check but must be
finite.  Each case prints the largest ratio of the two sides of the bound it measured.
"""
import ctypes
import functools
import math
from collections import OrderedDict

import numpy as np
import pytest
import torch

import di_engine_b200 as b2
from di_engine_b200 import ops
from oracle import rl_oracle
from tests import cases

pytestmark = pytest.mark.gpu
DEV = 'cuda'
K = 8.0
EPS32 = 2.0 ** -24
S_BIG = 128 * 512 + 37  # 256 full 256-row tiles and a ragged one: 257 tiles over 132 CTAs, one or two each (no ring wrap)
MASKS = {'1e8': -1e8, 'inf': -math.inf}
MIX_B = [0.7, 2.0, 0.05, -1.5]  # an upstream mix the forward pass does not expect


# ----------------------------------------------------------------------------------------------------------------
# generators
# ----------------------------------------------------------------------------------------------------------------
def _policy_pair(g, R, N, mask_val, scale_noise=(0.0, 0.05, 0.5, 2.0), regime_p=(0.2, 0.2, 0.3, 0.3)):
    """R rows of N logits: (new, old, action, regime, masked).  regime 0 on-policy (old is new bit for bit), 1 in band,
    2 clipped, 3 far off-policy.  ~20 % of the rows mask ~30 % of their non-chosen actions (some all of them) in both
    policies; ~10 % are scaled x8 (near-deterministic, a low-probability action is often the chosen one); every row is
    shifted by its own constant in [-50, 50]."""
    base = torch.randn(R, N, generator=g)
    sat = torch.rand(R, generator=g) < 0.1
    base[sat] *= 8.0
    regime = torch.multinomial(torch.tensor(regime_p), R, replacement=True, generator=g)
    action = torch.randint(0, N, (R, ), generator=g)
    noise = torch.tensor(scale_noise)[regime].unsqueeze(1) * torch.randn(R, N, generator=g)
    off = (torch.rand(R, 1, generator=g) * 100.0 - 50.0)
    new = base + off
    old = (base + noise) + off
    old[regime == 0] = new[regime == 0]
    mrow = torch.rand(R, generator=g) < 0.2
    mask = mrow.unsqueeze(1) & (torch.rand(R, N, generator=g) < 0.3)
    mask |= (mrow & (torch.rand(R, generator=g) < 0.15)).unsqueeze(1)  # only the chosen action left
    mask[torch.arange(R), action] = False
    new[mask] = mask_val
    old[mask] = mask_val
    return new, old, action, regime, mask


def _zeros_at(g, x, p):
    x = x.clone()
    x[torch.rand(x.shape, generator=g) < p] = 0.0
    return x


def ring_wrap_rows(N, pre=False, w=True, sms=None):
    """rows of a ppo_error batch on which the tile kernel's ring wraps: b200rl_ppo_tile_geometry on the device's SMs gives
    every CTA more 256-row tiles than its ring has stages, and the last tile is ragged"""
    if sms is None:
        sms = torch.cuda.get_device_properties(0).multi_processor_count
    lib = ops.lib()

    def geo(S):
        g = (ctypes.c_longlong * 3)()
        assert lib.b200rl_ppo_tile_geometry(S, N, int(pre), int(w), 0, sms, g) == 0
        return g[0], g[1]

    stages = geo(1 << 24)[1]
    S = sms * (stages + 1) * 256 + 37
    grid, st = geo(S)
    assert grid == sms and st == stages and (S // 256 + 1) // sms > stages, (N, pre, w, sms, grid, st)
    return S


def _samples(g, S, weight=True):
    t = {}
    t['value_new'] = torch.randn(S, generator=g)
    t['value_old'] = t['value_new'] + 0.3 * torch.randn(S, generator=g)
    t['adv'] = _zeros_at(g, torch.randn(S, generator=g), 0.05)
    t['return_'] = 2.0 * torch.randn(S, generator=g)
    t['weight'] = _zeros_at(g, torch.rand(S, generator=g), 0.05) if weight else None
    return t


def gen_ppo(seed, S, N, mask='1e8', A=None, weight=True, pretrained=False, **params):
    """ppo_error operands (S,) or (S, A) rows of N actions; returns (op, tensors, params, meta)."""
    g = cases._g(seed)
    rows = (S, ) if A is None else (S, A)
    R = int(np.prod(rows))
    new, old, action, regime, masked = _policy_pair(g, R, N, MASKS[mask])
    smp = _samples(g, S, weight)
    t = OrderedDict()
    t['logit_new'] = new.reshape(*rows, N)
    t['logit_old'] = old.reshape(*rows, N)
    t['action'] = action.reshape(rows)
    for k in ('value_new', 'value_old', 'adv', 'return_', 'weight'):
        t[k] = smp[k]
    t['logit_pretrained'] = None
    if pretrained:
        pre = new + 0.5 * torch.randn(R, N, generator=g)
        pre[masked] = MASKS[mask]
        t['logit_pretrained'] = pre.reshape(*rows, N)
    meta = dict(on=(regime == 0).reshape(rows), masked=masked.reshape(*rows, N))
    return 'ppo', t, dict(params), meta


def gen_cont(seed, S, D, factor=False, **params):
    """ppo_error_continuous / happo_error_continuous operands: mu_old = mu_new + 0.5 randn, sigma_old = sigma_new *
    exp(0.3 randn) off-policy, both identical in ~20 % of the samples; the action is drawn from the new policy."""
    g = cases._g(seed)
    t = OrderedDict()
    t['mu_new'] = torch.randn(S, D, generator=g)
    t['sigma_new'] = torch.exp(0.3 * torch.randn(S, D, generator=g))
    on = torch.rand(S, generator=g) < 0.2
    t['mu_old'] = torch.where(on.unsqueeze(1), t['mu_new'], t['mu_new'] + 0.5 * torch.randn(S, D, generator=g))
    t['sigma_old'] = torch.where(on.unsqueeze(1), t['sigma_new'],
                                 t['sigma_new'] * torch.exp(0.3 * torch.randn(S, D, generator=g)))
    t['action'] = t['mu_new'] + t['sigma_new'] * torch.randn(S, D, generator=g)
    for k, v in _samples(g, S).items():
        t[k] = v
    if factor:
        t['factor'] = torch.rand(S, 1, generator=g) * 2.7 + 0.3
        return 'happoc', t, dict(params), dict(on=on)
    t['mu_pretrained'] = t['sigma_pretrained'] = None
    return 'ppoc', t, dict(params), dict(on=on)


def gen_vtrace(seed, T, B, N, mask='1e8', **params):
    g = cases._g(seed)
    new, old, action, regime, masked = _policy_pair(g, T * B, N, MASKS[mask])
    t = OrderedDict()
    t['target_output'] = new.reshape(T, B, N)
    t['behaviour_output'] = old.reshape(T, B, N)
    t['action'] = action.reshape(T, B)
    t['value'] = torch.randn(T + 1, B, generator=g)
    t['reward'] = torch.rand(T, B, generator=g)
    t['weight'] = _zeros_at(g, torch.rand(T, B, generator=g), 0.05)
    return 'vtrace', t, dict(params), dict(on=(regime == 0).reshape(T, B), masked=masked.reshape(T, B, N))


def to64(t):
    return OrderedDict((k, v.double() if isinstance(v, torch.Tensor) and v.is_floating_point() else v)
                             for k, v in t.items())


# ----------------------------------------------------------------------------------------------------------------
# float64 per-sample terms: branch fractions, boundary rows and the scale of each signed loss
# ----------------------------------------------------------------------------------------------------------------
def _lp(logit, action):
    return cases._np(rl_oracle._chosen(rl_oracle._log_softmax_rows(logit.double()), action)).astype(np.float64)


def _value_terms(t, clip, use_value_clip):
    vn, vo, ret = (t[k].double().numpy() for k in ('value_new', 'value_old', 'return_'))
    dv = vn - vo
    e1 = (ret - vn) ** 2
    e2 = (ret - (vo + np.clip(dv, -clip, clip))) ** 2
    if not use_value_clip:
        return dict(), np.zeros(vn.shape, bool)
    bnd = (np.abs(np.abs(dv) - clip) <= 1e-5) | ((np.abs(dv) > clip) & (np.abs(e1 - e2) <= 1e-5 * np.maximum(e1, e2)))
    return dict(value_clipped=np.mean((np.abs(dv) > clip) & (e2 > e1))), bnd


def policy_terms(ratio, adv, w, fac, clip, dual_clip, dual_all=False):
    """fp64 ratio (S,) -> (branch fractions, boundary mask, sum of |selected surrogate * w| / S)."""
    lo, hi = float(np.float32(1 - clip)), float(np.float32(1 + clip))
    rc = np.clip(ratio, 1 - clip, 1 + clip)
    sel = np.minimum(ratio * adv, rc * adv) * fac
    bnd = (np.abs(ratio - lo) <= 1e-5 * lo) | (np.abs(ratio - hi) <= 1e-5 * hi)
    frac = dict(ratio_clipped=np.mean((ratio > hi) | (ratio < lo)))
    if dual_clip:
        where = np.ones_like(adv, bool) if dual_all else adv < 0
        floor = dual_clip * adv
        frac['dual_floor'] = np.mean(where & (sel < floor) & (adv < 0))
        near = (np.abs(fac * ratio - dual_clip) <= 1e-5 * dual_clip) | (np.abs(fac * rc - dual_clip) <= 1e-5 * dual_clip)
        bnd |= where & near
        sel = np.where(where, np.maximum(sel, floor), sel)
    return frac, bnd, np.mean(np.abs(sel) * w)


def ppo_meta(op, t, p, meta, adv=None):
    """branch fractions, boundary samples and loss scales of a ppo / ppo_policy / happo batch (float64)"""
    clip = p.get('clip_ratio', 0.2)
    lpn, lpo = _lp(t['logit_new'], t['action']), _lp(t['logit_old'], t['action'])
    ratio = np.exp(lpn - lpo)
    if ratio.ndim == 2:
        ratio = ratio.mean(1)
    adv = t['adv'].double().numpy() if adv is None else adv
    S = adv.shape[0]
    w = np.ones(S) if t['weight'] is None else t['weight'].double().numpy()
    fac = t['factor'].double().numpy().reshape(-1) if 'factor' in t else np.ones(S)
    frac, bnd, pol = policy_terms(ratio, adv, w, fac, clip, p.get('dual_clip'))
    scales = {'out_policy_loss': pol, 'out_approx_kl': np.mean(np.abs(lpo - lpn))}
    if 'value_new' in t:
        vf, vb = _value_terms(t, clip, p.get('use_value_clip', True))
        frac.update(vf)
        bnd |= vb
    if t.get('logit_pretrained') is not None:
        scales['out_kl_div'] = np.mean(np.abs(lpn - _lp(t['logit_pretrained'], t['action'])))
    frac['on_policy'] = float(meta['on'].double().mean())
    frac['masked_rows'] = float(meta['masked'].any(-1).double().mean())
    assert np.abs(lpn - lpo).max() < 60, 'fp32 ratio would overflow'
    return frac, bnd, scales


def check_branches(frac, need):
    for k in need:
        assert frac[k] >= 0.02, ('generator does not reach branch', k, frac)


# ----------------------------------------------------------------------------------------------------------------
# the comparison rule
# ----------------------------------------------------------------------------------------------------------------
def compare64(tag, got, r32, r64, scales=None, bnd=None, S=None):
    """max|gpu - fp64| <= K * max(max|fp32 - fp64|, 2^-24 * scale) for every output; returns the largest ratio."""
    scales = scales or {}
    worst, worst_k = 0.0, None
    n_bnd = 0 if bnd is None else int(bnd.sum())
    if bnd is not None:
        assert n_bnd <= 1e-3 * bnd.size, (tag, 'boundary rows', n_bnd)
    assert set(got) == set(r64), (sorted(got), sorted(r64))
    for k in r64:
        x, a, b = (np.asarray(d[k], np.float64) for d in (got, r32, r64))
        assert x.shape == b.shape, (tag, k, x.shape, b.shape)
        fin = np.isfinite(b)
        assert np.array_equal(np.isnan(x[~fin]), np.isnan(b[~fin])), (tag, k, 'non-finite pattern')
        assert np.isfinite(x[fin]).all(), (tag, k, 'NaN / inf where the fp64 reference is finite')
        if k == 'out_clipfrac':
            assert abs(float(x) - float(b)) * S <= n_bnd + 0.5, (tag, k, float(x), float(b), n_bnd)
            continue
        keep = fin
        if k.startswith('grad_'):
            scale = float(np.abs(b[fin]).max()) if fin.any() else 0.0
            if bnd is not None and bnd.shape[0] == b.shape[0]:
                keep = fin & ~bnd.reshape((-1, ) + (1, ) * (b.ndim - 1))
        else:
            scale = float(scales.get(k, np.abs(b[fin]).max() if fin.any() else 0.0))
        if not keep.any():
            continue
        e_gpu = float(np.abs(x - b)[keep].max())
        # where the fp32 oracle itself overflows (finfo.min * a large upstream gradient at a -inf logit) only the fp64
        # scale bounds the error
        e32 = np.abs(a - b)[keep & np.isfinite(a)]
        e32 = float(e32.max()) if e32.size else 0.0
        floor = max(e32, EPS32 * scale)
        ratio = e_gpu / floor if floor > 0 else (0.0 if e_gpu == 0 else math.inf)
        assert e_gpu <= K * floor, (tag, k, 'err_gpu %.3e  err_fp32 %.3e  2^-24*scale %.3e  ratio %.2f' % (
            e_gpu, e32, EPS32 * scale, ratio))
        if ratio >= worst:
            worst, worst_k = ratio, k
    print('\n[fp64] %-48s max err_gpu/bound_floor %.2f (%s)  boundary rows %d' % (tag, worst, worst_k, n_bnd))
    return worst


def zero_at_masked(tag, got, key, masked):
    g = np.asarray(got[key])
    assert np.all(g[masked] == 0.0), (tag, key, 'gradient at masked entries', float(np.abs(g[masked]).max()))


# ----------------------------------------------------------------------------------------------------------------
# reference + GPU runs with a chosen upstream mix
# ----------------------------------------------------------------------------------------------------------------
class _Mix:
    def __init__(self, op, mix):
        self.op, self.mix = op, list(mix)

    def __enter__(self):
        self.old = cases.LOSS_MIX[self.op]
        cases.LOSS_MIX[self.op] = self.mix

    def __exit__(self, *exc):
        cases.LOSS_MIX[self.op] = self.old


def mixes(op):
    a = cases.LOSS_MIX[op]
    return a, MIX_B[:len(a)]


def refs(op, t, p, mix, runner=None):
    run = runner or (lambda tt: cases.run_oracle(rl_oracle, op, tt, p))
    with _Mix(op, mix):
        return run(t), run(to64(t))


def gpu_paths(op, run_gpu, mix_a, mix_b):
    """the same batch through the forward-written gradients (expected mix) and the recompute launch (unexpected mix):
    yields (path, mix, result)"""
    with _Mix(op, mix_a):
        run_gpu()  # the backward records mix_a as the expectation of the next forward
        yield 'expected', 0, run_gpu()
    with _Mix(op, mix_b):
        yield 'unexpected', 1, run_gpu()


def run_gpu_api(op, t, p):
    return lambda: cases.run_api(b2.rl_utils, op, t, p, device=DEV)


# ----------------------------------------------------------------------------------------------------------------
# ppo_error: tile kernel (N <= 32: compile-time N, generic N, ragged tail), thread-per-row (N 33..64, multi-agent,
# unaligned) and warp-per-row (N > 64) fallbacks; fused and separate backward
# ----------------------------------------------------------------------------------------------------------------
PPO_CASES = {
    'N2': dict(S=S_BIG, N=2, weight=False),
    'N6_dc': dict(S=S_BIG, N=6, dual_clip=3.0),
    'N11': dict(S=S_BIG, N=11),
    'N18_dc': dict(S=S_BIG, N=18, dual_clip=3.0),
    'N32_dc': dict(S=S_BIG, N=32, dual_clip=3.0),
    'N40_dc': dict(S=4099, N=40, dual_clip=3.0),
    'N100': dict(S=2053, N=100),
    'marl_A4_N7_dc': dict(S=3001, N=7, A=4, dual_clip=3.0),
    'odd_offset_N6_dc': dict(S=4099, N=6, dual_clip=3.0, odd=True),
    'pre_k1_N6': dict(S=S_BIG, N=6, pretrained=True, kl_type='k1'),
    'pre_k2_N18_dc': dict(S=4099, N=18, pretrained=True, kl_type='k2', dual_clip=3.0),
    'pre_k3_N13': dict(S=4099, N=13, pretrained=True, kl_type='k3'),
    'ring_wrap_N6_dc': dict(S='wrap', N=6, dual_clip=3.0),  # every CTA runs its 8-stage ring more than once
}


def _odd(x):
    """a device copy of ``x`` that starts 4 bytes into its storage: not 16-byte aligned"""
    buf = torch.zeros(x.numel() + 1, dtype=x.dtype, device=DEV)
    buf[1:].copy_(x.reshape(-1))
    return buf[1:].view(x.shape)


def _run_ppo_odd(t, p):
    td = OrderedDict((k, None if v is None else _odd(v)) for k, v in t.items())
    for k in cases.GRAD_INPUTS['ppo']:
        td[k].requires_grad_(True)
    assert td['logit_new'].data_ptr() % 16 != 0
    data = b2.ppo_data(*[td[k] for k in ('logit_new', 'logit_old', 'action', 'value_new', 'value_old', 'adv', 'return_',
                                         'weight', 'logit_pretrained')])
    loss, info = b2.ppo_error(data, **p)
    res = OrderedDict(('out_' + k, cases._np(getattr(loss, k))) for k in ('policy_loss', 'value_loss', 'entropy_loss',
                                                                                  'kl_div'))
    res['out_approx_kl'], res['out_clipfrac'] = np.float32(info.approx_kl), np.float32(info.clipfrac)
    cases._backward('ppo', list(loss), td, res)
    return res


@functools.lru_cache(maxsize=4)
def _ppo_batch(name, mask):
    c = dict(PPO_CASES[name])
    S, N, odd = c.pop('S'), c.pop('N'), c.pop('odd', False)
    if S == 'wrap':
        S = ring_wrap_rows(N, c.get('pretrained', False), c.get('weight', True))
    op, t, p, meta = gen_ppo(7000 + list(PPO_CASES).index(name), S, N, mask=mask, clip_ratio=0.2, **c)
    frac, bnd, scales = ppo_meta(op, t, p, meta)
    a, b = mixes(op)
    return op, t, p, meta, frac, bnd, scales, odd, (refs(op, t, p, a), refs(op, t, p, b))


@pytest.mark.parametrize('backward', ['fused', 'separate'])
@pytest.mark.parametrize('mask', sorted(MASKS))
@pytest.mark.parametrize('name', list(PPO_CASES))
def test_ppo_error_fp64(name, mask, backward):
    op, t, p, meta, frac, bnd, scales, odd, rr = _ppo_batch(name, mask)
    check_branches(frac, ['ratio_clipped', 'value_clipped', 'on_policy', 'masked_rows'] +
                   (['dual_floor'] if p.get('dual_clip') else []))
    run = (lambda: _run_ppo_odd(t, p)) if odd else run_gpu_api(op, t, p)
    ops.PPO_FUSED_BACKWARD = backward == 'fused'
    try:
        for path, i, got in gpu_paths(op, run, *mixes(op)):
            tag = 'ppo %s %s %s %s' % (name, mask, backward, path)
            compare64(tag, got, *rr[i], scales=scales, bnd=bnd, S=len(bnd))
            zero_at_masked(tag, got, 'grad_logit_new', meta['masked'].numpy())
    finally:
        ops.PPO_FUSED_BACKWARD = True
    print('[fp64] branches %s %s' % (name, {k: round(float(v), 3) for k, v in frac.items()}))


# ----------------------------------------------------------------------------------------------------------------
# gae -> ppo_error in one launch: row tiles (fused.cu) and column tiles (colws.cu)
# ----------------------------------------------------------------------------------------------------------------
GAE_PPO_SHAPES = [(128, 4096, 6, 3.0), (64, 260, 18, None), (33, 20, 11, 3.0)]


@functools.lru_cache(maxsize=2)
def _gae_ppo_batch(shape, mask):
    T, B, N, dc = shape
    _, tg, pg = cases.gae_case(7100 + T, T, B, p_done=0.03, gamma=0.99, lambda_=0.95)
    op, tp, p, meta = gen_ppo(7200 + T, T * B, N, mask=mask, clip_ratio=0.2, dual_clip=dc)
    og = {k: v.clone() for k, v in tg.items()}
    adv = rl_oracle.gae(og['value'], og['next_value'], og['reward'], og['done'], og['traj_flag'], **pg)
    tp['adv'] = adv.reshape(-1)  # the fp32 advantage feeds both references: the kernel must reproduce it bit for bit
    frac, bnd, scales = ppo_meta(op, tp, p, meta)
    a, b = mixes(op)
    return tg, pg, og['next_value'], adv, tp, p, meta, frac, bnd, scales, (refs(op, tp, p, a), refs(op, tp, p, b))


def _run_gae_ppo(tg, pg, tp, p, nv_want, adv_want):
    dg = {k: v.clone().to(DEV) for k, v in tg.items()}
    td = cases.prepare('ppo', tp, DEV)
    adv, loss, info = b2.gae_ppo_error(
        b2.gae_data(dg['value'], dg['next_value'], dg['reward'], dg['done'], dg['traj_flag']),
        b2.ppo_data(td['logit_new'], td['logit_old'], td['action'], td['value_new'], td['value_old'], None, td['return_'],
                    td['weight'], td['logit_pretrained']), pg['gamma'], pg['lambda_'], **p)
    assert torch.equal(adv.cpu(), adv_want) and torch.equal(dg['next_value'].cpu(), nv_want)
    res = OrderedDict(('out_' + k, cases._np(getattr(loss, k))) for k in ('policy_loss', 'value_loss', 'entropy_loss',
                                                                                  'kl_div'))
    res['out_approx_kl'], res['out_clipfrac'] = np.float32(info.approx_kl), np.float32(info.clipfrac)
    cases._backward('ppo', list(loss), td, res)
    return res


@pytest.mark.parametrize('impl', ['row', 'col'])
@pytest.mark.parametrize('mask', sorted(MASKS))
@pytest.mark.parametrize('shape', GAE_PPO_SHAPES, ids=lambda s: '%dx%dx%d' % s[:3])
def test_gae_ppo_error_fp64(shape, mask, impl):
    tg, pg, nv, adv, tp, p, meta, frac, bnd, scales, rr = _gae_ppo_batch(shape, mask)
    check_branches(frac, ['ratio_clipped', 'value_clipped', 'on_policy', 'masked_rows'] +
                   (['dual_floor'] if p.get('dual_clip') else []))
    old = ops.lib().b200rl_gae_ppo_set_impl({'row': 1, 'col': 2}[impl])
    try:
        for path, i, got in gpu_paths('ppo', lambda: _run_gae_ppo(tg, pg, tp, p, nv, adv), *mixes('ppo')):
            tag = 'gae_ppo %s %s %s %s' % ('x'.join(map(str, shape[:3])), mask, impl, path)
            compare64(tag, got, *rr[i], scales=scales, bnd=bnd, S=len(bnd))
            zero_at_masked(tag, got, 'grad_logit_new', meta['masked'].numpy())
    finally:
        ops.lib().b200rl_gae_ppo_set_impl(old)
    print('[fp64] branches gae_ppo %s %s' % (shape[:3], {k: round(float(v), 3) for k, v in frac.items()}))


# ----------------------------------------------------------------------------------------------------------------
# the other PPO-family operators on the generator batch
# ----------------------------------------------------------------------------------------------------------------
def _adv_norm_runner(p, device):
    def run(t):
        tt = cases.prepare('ppo', t, device)
        res = OrderedDict()
        if device == 'cpu':
            tt['adv'] = rl_oracle.normalize_advantage(tt['adv'])
            out = rl_oracle.ppo_error(**tt, **p)
            loss, akl, cf = out[:4], out[4], out[5]
        else:
            data = b2.ppo_data(*[tt[k] for k in ('logit_new', 'logit_old', 'action', 'value_new', 'value_old', 'adv',
                                                 'return_', 'weight', 'logit_pretrained')])
            loss, info = b2.ppo_error_adv_norm(data, **p)
            akl, cf = info.approx_kl, info.clipfrac
        for k, v in zip(('policy_loss', 'value_loss', 'entropy_loss', 'kl_div'), loss):
            res['out_' + k] = cases._np(v)
        res['out_approx_kl'], res['out_clipfrac'] = np.float32(akl), np.float32(cf)
        cases._backward('ppo', list(loss), tt, res)
        return res
    return run


def _family_case(kind, mask):
    """(op, tensors, params, meta, runner for the references or None, the fp64 advantage the loss sees)"""
    if kind == 'adv_norm':
        op, t, p, meta = gen_ppo(7301, 4099, 6, mask=mask, clip_ratio=0.2, dual_clip=3.0)
        t['adv'] = t['adv'] * 3.0 + 0.7
        return op, t, p, meta, _adv_norm_runner(p, 'cpu'), rl_oracle.normalize_advantage(t['adv'].double()).numpy()
    if kind in ('policy_ent', 'policy_noent'):
        op, t, p, meta = gen_ppo(7302, 4099, 6, mask=mask, clip_ratio=0.2, dual_clip=3.0)
        t = OrderedDict((k, t[k]) for k in ('logit_new', 'logit_old', 'action', 'adv', 'weight', 'logit_pretrained'))
        p['entropy_bonus'] = kind == 'policy_ent'
        return 'ppo_policy', t, p, meta, None, None
    if kind == 'happo':
        op, t, p, meta = gen_ppo(7303, 4099, 6, mask=mask, clip_ratio=0.2, dual_clip=3.0)
        t = OrderedDict((k, t[k]) for k in cases.HAPPO_FIELDS if k != 'factor')
        t['factor'] = torch.rand(4099, 1, generator=cases._g(7304)) * 2.7 + 0.3  # factor * min crosses the floor both ways
        return 'happo', t, p, meta, None, None
    if kind == 'ppg':
        op, t, p, meta = gen_ppo(7305, 4099, 6, mask=mask, clip_ratio=0.2)
        t = OrderedDict((k, t[k]) for k in ('logit_new', 'logit_old', 'action', 'value_new', 'value_old', 'return_',
                                                  'weight'))
        return 'ppg', t, p, meta, None, None
    raise KeyError(kind)


@pytest.mark.parametrize('mask', sorted(MASKS))
@pytest.mark.parametrize('kind', ['adv_norm', 'policy_ent', 'policy_noent', 'happo', 'ppg'])
def test_ppo_family_fp64(kind, mask):
    op, t, p, meta, runner, adv64 = _family_case(kind, mask)
    mix_op = 'ppo' if kind == 'adv_norm' else op
    if op == 'ppg':  # no surrogate: only the value clip branches
        frac, bnd = _value_terms(t, p['clip_ratio'], True)
        frac['masked_rows'] = float(meta['masked'].any(-1).double().mean())
        scales, need = {}, ['value_clipped', 'masked_rows']
    else:
        frac, bnd, scales = ppo_meta(op, t, p, meta, adv=adv64)
        need = ['ratio_clipped', 'dual_floor', 'on_policy', 'masked_rows'] + (['value_clipped'] if 'value_new' in t else [])
    check_branches(frac, need)
    a, b = mixes(mix_op)
    rr = (refs(mix_op, t, p, a, runner), refs(mix_op, t, p, b, runner))
    run = _adv_norm_runner(p, DEV) if kind == 'adv_norm' else None
    for path, i, got in gpu_paths(mix_op, (lambda: run(t)) if run else run_gpu_api(op, t, p), a, b):
        tag = '%s %s %s' % (kind, mask, path)
        compare64(tag, got, *rr[i], scales=scales, bnd=bnd, S=len(bnd))
        zero_at_masked(tag, got, 'grad_logit_new', meta['masked'].numpy())
    print('[fp64] branches %s %s' % (kind, {k: round(float(v), 3) for k, v in frac.items()}))


def test_ppo_value_error_fp64():
    op, t, p, meta = gen_ppo(7306, 70001, 2, clip_ratio=0.2)
    t = OrderedDict((k, t[k]) for k in ('value_new', 'value_old', 'return_', 'weight'))
    frac, bnd = _value_terms(t, 0.2, True)
    check_branches(frac, ['value_clipped'])
    for mix in ([0.7], [2.0]):
        r32, r64 = refs('ppo_value', t, p, mix)
        with _Mix('ppo_value', mix):
            got = cases.run_api(b2.rl_utils, 'ppo_value', t, p, device=DEV)
        compare64('ppo_value mix %s' % mix, got, r32, r64, bnd=bnd, S=len(bnd))


# ----------------------------------------------------------------------------------------------------------------
# continuous-action PPO / HAPPO (heads.cu ppoc_kernel: the dual clip applies to every sample)
# ----------------------------------------------------------------------------------------------------------------
def cont_meta(op, t, p):
    mu, sg, mo, so, act = (t[k].double() for k in ('mu_new', 'sigma_new', 'mu_old', 'sigma_old', 'action'))

    def logp(m, s):
        return -((act - m) ** 2) / (2 * s ** 2) - s.log() - math.log(math.sqrt(2 * math.pi))

    d = (logp(mu, sg) - logp(mo, so)).numpy()
    ratio = np.exp(d.sum(-1))
    adv, w = t['adv'].double().numpy(), t['weight'].double().numpy()
    fac = t['factor'].double().numpy().reshape(-1) if 'factor' in t else np.ones_like(adv)
    # both operators apply max(factor * min(...), dual * adv) to every sample
    frac, bnd, pol = policy_terms(ratio, adv, w, fac, p['clip_ratio'], p['dual_clip'], dual_all=True)
    vf, vb = _value_terms(t, p['clip_ratio'], True)
    frac.update(vf)
    assert np.abs(d.sum(-1)).max() < 60
    akl = np.mean(np.abs(d)) if op == 'happoc' else np.mean(np.abs(d.sum(-1)))
    return frac, bnd | vb, {'out_policy_loss': pol, 'out_approx_kl': akl}


@pytest.mark.parametrize('op_kind', ['ppoc', 'happoc'])
def test_continuous_ppo_fp64(op_kind):
    op, t, p, meta = gen_cont(7400 + len(op_kind), 4099, 3, factor=op_kind == 'happoc', clip_ratio=0.2, dual_clip=3.0)
    frac, bnd, scales = cont_meta(op, t, p)
    frac['on_policy'] = float(meta['on'].double().mean())
    check_branches(frac, ['ratio_clipped', 'dual_floor', 'value_clipped', 'on_policy'])
    a, b = mixes(op)
    rr = (refs(op, t, p, a), refs(op, t, p, b))
    for path, i, got in gpu_paths(op, run_gpu_api(op, t, p), a, b):
        compare64('%s %s' % (op, path), got, *rr[i], scales=scales, bnd=bnd, S=len(bnd))
    print('[fp64] branches %s %s' % (op, {k: round(float(v), 3) for k, v in frac.items()}))


# ----------------------------------------------------------------------------------------------------------------
# a2c_error (heads.cu a2c_kernel)
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('mask', sorted(MASKS))
def test_a2c_error_fp64(mask):
    _, tp, _, meta = gen_ppo(7500, 4099, 6, mask=mask)
    t = OrderedDict([('logit', tp['logit_new']), ('action', tp['action']), ('value', tp['value_new']),
                           ('adv', tp['adv']), ('return_', tp['return_']), ('weight', tp['weight'])])
    assert float(meta['masked'].any(-1).double().mean()) >= 0.02
    lp = _lp(t['logit'], t['action'])
    scales = {'out_policy_loss': np.mean(np.abs(lp * t['adv'].double().numpy() * t['weight'].double().numpy()))}
    a, b = mixes('a2c')
    rr = (refs('a2c', t, {}, a), refs('a2c', t, {}, b))
    for path, i, got in gpu_paths('a2c', run_gpu_api('a2c', t, {}), a, b):
        tag = 'a2c %s %s' % (mask, path)
        compare64(tag, got, *rr[i], scales=scales)
        zero_at_masked(tag, got, 'grad_logit', meta['masked'].numpy())


# ----------------------------------------------------------------------------------------------------------------
# V-trace: vtws.cu (streaming and resident one-launch kernels) and the pg.cu tiles / fallbacks
# ----------------------------------------------------------------------------------------------------------------
VT_PARAMS = dict(gamma=0.99, lambda_=0.95, rho_clip_ratio=0.9, c_clip_ratio=1.1, rho_pg_clip_ratio=1.3)


def vtrace_scales(t, p):
    """fp64 |lp * adv * w| mean (the policy loss' per-sample terms), with the reference's own V-trace targets"""
    tt = to64(t)
    lp_t = torch.from_numpy(_lp(tt['target_output'], tt['action']))
    isw = torch.exp(lp_t - torch.from_numpy(_lp(tt['behaviour_output'], tt['action'])))
    v, r, g = tt['value'], tt['reward'], p['gamma']
    rho, cs = isw.clamp(max=p['rho_clip_ratio']), isw.clamp(max=p['c_clip_ratio'])
    deltas = rho * (r + g * v[1:] - v[:-1])
    vs, carry = v[:-1].clone(), 0.
    for i in range(r.shape[0] - 1, -1, -1):
        carry = deltas[i] + g * p['lambda_'] * cs[i] * carry
        vs[i] += carry
    adv = isw.clamp(max=p['rho_pg_clip_ratio']) * (r + g * torch.cat([vs[1:], v[-1:]], 0) - v[:-1])
    frac = dict(is_far_above=float((isw > 2 * p['rho_clip_ratio']).double().mean()),
                is_far_below=float((isw < 0.5 * p['rho_clip_ratio']).double().mean()))
    return {'out_policy_loss': float((lp_t * adv * tt['weight']).abs().mean())}, frac


@functools.lru_cache(maxsize=2)
def _vt_batch(shape, mask):
    T, B, N = shape
    op, t, p, meta = gen_vtrace(7600 + T + N, T, B, N, mask=mask, **VT_PARAMS)
    scales, frac = vtrace_scales(t, p)
    frac['on_policy'] = float(meta['on'].double().mean())
    frac['masked_rows'] = float(meta['masked'].any(-1).double().mean())
    a, b = mixes(op)
    return op, t, p, meta, scales, frac, (refs(op, t, p, a), refs(op, t, p, b))


@pytest.mark.parametrize('impl', ['auto', 'resident', 'pg'])
@pytest.mark.parametrize('mask', sorted(MASKS))
@pytest.mark.parametrize('shape', [(64, 8192, 6), (33, 20, 11), (24, 64, 18), (8, 16, 100)], ids=lambda s: '%dx%dx%d' % s)
def test_vtrace_fp64(shape, mask, impl):
    op, t, p, meta, scales, frac, rr = _vt_batch(shape, mask)
    check_branches(frac, ['is_far_above', 'is_far_below', 'on_policy', 'masked_rows'])
    old = ops.lib().b200rl_vtrace_set_impl({'auto': 0, 'resident': 2, 'pg': 0}[impl])
    ops.VTRACE_FUSED = impl != 'pg'
    try:
        for path, i, got in gpu_paths(op, run_gpu_api(op, t, p), *mixes(op)):
            tag = 'vtrace %s %s %s %s' % ('x'.join(map(str, shape)), mask, impl, path)
            compare64(tag, got, *rr[i], scales=scales)
            zero_at_masked(tag, got, 'grad_target_output', meta['masked'].numpy())
    finally:
        ops.VTRACE_FUSED = True
        ops.lib().b200rl_vtrace_set_impl(old)
        ops.vtrace_hint(torch.device(DEV)).copy_(torch.tensor(cases.LOSS_MIX['vtrace']))
    print('[fp64] branches vtrace %s %s' % (shape, {k: round(float(v), 3) for k, v in frac.items()}))


# ----------------------------------------------------------------------------------------------------------------
# the tile kernels' entropy factor with a large entropy coefficient and a -inf logit: |g_ent * w * ln2 / S| > 1
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('path', ['ppo', 'vtrace'])
def test_tile_entropy_factor_with_minus_inf_logit(path):
    """2 rows, weight 4, entropy upstream gradient 1: k1 = 1 * 4 * ln2 / 2 > 1.  ppo_error N = 6 runs the PPO tile kernel;
    V-trace at B = 2 runs the pg.cu tiles (the one-launch kernels need B % 4 == 0).  The fp32 oracle overflows here itself
    (its entropy backward multiplies finfo.min by 2): the fp64 reference is finite."""
    g = cases._g(7700)
    if path == 'ppo':
        op, t, p, meta = gen_ppo(7701, 2, 6, weight=True)
        t['logit_new'] = torch.randn(2, 6, generator=g)
        t['logit_old'] = t['logit_new'] + 0.5 * torch.randn(2, 6, generator=g)
        t['action'] = torch.tensor([1, 4])
        t['weight'] = torch.full((2, ), 4.0)
        for k in ('logit_new', 'logit_old'):
            t[k][0, 3] = -math.inf
        mix, gkey = [1.0, 0.5, 1.0, 0.0], 'grad_logit_new'
    else:
        op, t, p, meta = gen_vtrace(7702, 1, 2, 6, **VT_PARAMS)
        t['target_output'] = torch.randn(1, 2, 6, generator=g)
        t['behaviour_output'] = t['target_output'] + 0.5 * torch.randn(1, 2, 6, generator=g)
        t['action'] = torch.tensor([[1, 4]])
        t['weight'] = torch.full((1, 2), 4.0)
        for k in ('target_output', 'behaviour_output'):
            t[k][0, 0, 3] = -math.inf
        mix, gkey = [1.0, 0.5, 1.0], 'grad_target_output'
    r32, r64 = refs(op, t, p, mix)
    ops.VTRACE_FUSED = False
    try:
        for _, _, got in gpu_paths(op, run_gpu_api(op, t, p), mix, mix):
            compare64('entropy factor %s' % path, got, r32, r64, S=2)
            assert np.asarray(got[gkey]).reshape(2, 6)[0, 3] == 0.0
    finally:
        ops.VTRACE_FUSED = True
        ops.vtrace_hint(torch.device(DEV)).copy_(torch.tensor(cases.LOSS_MIX['vtrace']))
        ops.ppo_hint(torch.device(DEV)).copy_(torch.tensor([1.0, 0.5, -0.01, 0.0]))


# ----------------------------------------------------------------------------------------------------------------
# exact ties: clip_ratio 0.25 and values on a 2^-10 grid, so every subtraction in the value clip is exact
# ----------------------------------------------------------------------------------------------------------------
def tie_batch(S, N, A=None, on_policy_only=False):
    g = cases._g(7800 + N)
    rows = (S, ) if A is None else (S, A)
    t = OrderedDict()
    t['logit_new'] = torch.randn(*rows, N, generator=g)
    t['logit_old'] = t['logit_new'].clone()
    if not on_policy_only:
        off = torch.rand(S, generator=g) < 0.5
        t['logit_old'][off] += 0.5 * torch.randn(int(off.sum()), *rows[1:], N, generator=g)
    t['action'] = torch.randint(0, N, rows, generator=g)
    q = 1.0 / 1024
    t['value_new'] = torch.randint(-2048, 2048, (S, ), generator=g).float() * q
    sign = torch.randint(0, 2, (S, ), generator=g).float() * 2 - 1
    kind = torch.randint(0, 3, (S, ), generator=g)  # dv = +-clip exactly, inside, outside
    dv = torch.where(kind == 0, 0.25 * sign, torch.where(kind == 1, 0.125 * sign, 0.5 * sign))
    t['value_old'] = t['value_new'] - dv
    t['adv'] = torch.randn(S, generator=g)
    t['adv'][torch.rand(S, generator=g) < 0.3] = 0.0
    t['return_'] = torch.randint(-4096, 4096, (S, ), generator=g).float() * q
    t['weight'] = torch.randint(0, 1025, (S, ), generator=g).float() * q
    t['logit_pretrained'] = None
    assert torch.equal(t['value_new'] - t['value_old'], dv)
    return t


@pytest.mark.parametrize('where', ['tile_N6', 'thread_N40', 'warp_N100', 'marl_A3_N5', 'gae_ppo_row', 'gae_ppo_col',
                                   'happo', 'ppo_policy'])
def test_exact_ties_and_on_policy_batch(where):
    N = {'thread_N40': 40, 'warp_N100': 100, 'marl_A3_N5': 5}.get(where, 6)
    A = 3 if where == 'marl_A3_N5' else None
    p = dict(clip_ratio=0.25, dual_clip=3.0)
    for on_only in (False, True):
        S = 4096 if where.startswith('gae') else 1031
        t = tie_batch(S, N, A, on_policy_only=on_only)
        op = 'ppo'
        if where == 'happo':
            op = 'happo'
            t = OrderedDict((k, t[k]) for k in cases.HAPPO_FIELDS if k != 'factor')
            t['factor'] = torch.randint(256, 2048, (S, 1), generator=cases._g(7899)).float() / 1024
        elif where == 'ppo_policy':
            op = 'ppo_policy'
            t = OrderedDict((k, t[k]) for k in ('logit_new', 'logit_old', 'action', 'adv', 'weight', 'logit_pretrained'))
        mix = cases.LOSS_MIX[op]
        r32, r64 = refs(op, t, p, mix)
        if where.startswith('gae'):
            T, B = 64, 64
            _, tg, pg = cases.gae_case(7890, T, B, p_done=0.03)
            og = {k: v.clone() for k, v in tg.items()}
            adv = rl_oracle.gae(og['value'], og['next_value'], og['reward'], og['done'], og['traj_flag'], **pg)
            t['adv'] = adv.reshape(-1)
            r32, r64 = refs(op, t, p, mix)
            old = ops.lib().b200rl_gae_ppo_set_impl(1 if where.endswith('row') else 2)
            try:
                with _Mix(op, mix):
                    got = _run_gae_ppo(tg, pg, t, p, og['next_value'], adv)
            finally:
                ops.lib().b200rl_gae_ppo_set_impl(old)
        else:
            with _Mix(op, mix):
                got = cases.run_api(b2.rl_utils, op, t, p, device=DEV)
        compare64('ties %s on_policy_only=%s' % (where, on_only), got, r32, r64, bnd=np.zeros(S, bool), S=S)
        if on_only:
            assert float(got['out_approx_kl']) == 0.0 and float(got['out_clipfrac']) == 0.0, (where, got['out_approx_kl'])


def test_continuous_on_policy_batch_is_exactly_on_policy():
    op, t, p, meta = gen_cont(7900, 1031, 3, clip_ratio=0.25, dual_clip=3.0)
    t['mu_old'], t['sigma_old'] = t['mu_new'].clone(), t['sigma_new'].clone()
    got = cases.run_api(b2.rl_utils, op, t, p, device=DEV)
    assert float(got['out_approx_kl']) == 0.0 and float(got['out_clipfrac']) == 0.0
