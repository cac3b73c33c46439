"""The batch statistics around gae against a float64 reference, on offset-heavy, degenerate and non-finite batches.

PPOPolicy and PPOFPolicy compute two sets of statistics around every advantage recompute, and divide every advantage of the
batch by one of them:

* ``return_stats`` {mean, np.var, count} of the unnormalised return (``gae_returns``) or of the stored return
  (``ppof_gae_returns(..., 'baseline')``) -- what ``RunningMeanStd.update`` receives;
* ``adv_stats`` {adv.mean(), adv.std() + 1e-8} (``gae_returns``, ``ppof_gae_returns``, ``normalize_advantage``,
  ``ppo_error_adv_norm``).

The parity suites draw ``randn``-like batches, where the mean is comparable to the spread.  Here the batches sit 1e2 to 1e6
standard deviations away from 0 (returns of a constant per-step reward over a long horizon; advantages of a converged critic
with a constant bias), are constant, two-valued, tiny, subnormal, near fp32's largest value, or hold inf / NaN.

Reference: the statistics describe fp32 tensors the kernels themselves write; those tensors are first pinned bit for bit to
``rl_oracle``.  The float64 reference is numpy / torch on float64 copies of them; the yardstick is the fp32 computation the
learner would run (``np.mean`` / ``np.var`` on the fp32 array, torch fp32 ``mean`` / ``std`` on the same CUDA tensor).  Every
output obeys ``test_offpolicy_fp64.compare64``'s rule with its K = 8.  Every multi-CTA case runs three times on the same
inputs and workspace and must give the same bits.

The fp32 yardstick loosens as the offset grows: ``np.var`` on the fp32 array subtracts a mean rounded to fp32, so past about
1e5 sd its error is a visible fraction of the variance and fp64 sums with plain cancellation still fit inside K times it.
The accuracy of the return variance is therefore pinned by the 1e2 - 1e4 offsets, the constant batches, and the batches
whose offset sits in the value (the 'voff' regimes: the advantage is centred, the return is not) under value_norm scales far
from 1, where a return statistic taken around anything but a member of the batch fails.  The larger offsets pin the fixed
order of the join (the repeats) and the mean.
"""
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
from tests.test_offpolicy_fp64 import _adv_norm_runner, compare64, gen_ppo, mixes, ppo_meta, refs

DEV = 'cuda'
GAMMA, LAMBDA = 0.99, 0.95
VN_STD = 1.7320508  # bench.py's value_norm std
ADV_SPREAD = math.sqrt(1.0 / (1.0 - (GAMMA * LAMBDA)**2))  # sd of sum_k f^k z_k over the sd of z
F32_MAX = float(np.finfo(np.float32).max)


# ----------------------------------------------------------------------------------------------------------------
# float64 reference and fp32 yardstick
# ----------------------------------------------------------------------------------------------------------------
def pop_stats64(x):
    """RunningMeanStd.update's {mean, np.var, count} of an fp32 array, in float64"""
    x = np.asarray(x, np.float32).reshape(-1).astype(np.float64)
    with np.errstate(all='ignore'):
        return OrderedDict(mean=np.mean(x), var=np.var(x), count=float(x.size))


def pop_stats32(x):
    """the same in fp32, as the learner computes it from the array it copies to the host"""
    x = np.asarray(x, np.float32).reshape(-1)
    with np.errstate(all='ignore'):
        return OrderedDict(mean=np.mean(x), var=np.var(x), count=float(x.size))


def adv_stats_ref(x):
    """{adv.mean(), adv.std() + 1e-8} (policy/ppo.py:304-306) of a torch tensor, in its own precision"""
    return OrderedDict(mean=x.mean().item(), std=(x.std() + 1e-8).item())


def check_stats(tag, got, r32, r64, ppo_var_clamp=False):
    """compare64 on the finite outputs; a float64 value beyond fp32's range must come back as that infinity, a non-finite
    one as the same non-finite value, the count exactly.  ``ppo_var_clamp``: the PPO build clamps a NaN variance to 0."""
    got = OrderedDict((k, float(v)) for k, v in got.items())
    r64 = OrderedDict((k, float(v)) for k, v in r64.items())
    if ppo_var_clamp and 'var' in r64 and math.isnan(r64['var']):
        r64['var'] = 0.0
    if 'count' in r64:
        assert got.pop('count') == r64.pop('count'), (tag, 'count')
    fin = OrderedDict()
    for k in r64:
        want = r64[k]
        if math.isfinite(want) and abs(want) > F32_MAX:  # rounds to +-inf in fp32
            want = math.copysign(math.inf, want)
        if math.isfinite(want):
            fin[k] = want
        else:
            assert got[k] == want or (math.isnan(got[k]) and math.isnan(want)), (tag, k, got[k], want)
    if not fin:
        return 0.0
    return compare64(tag, OrderedDict((k, got[k]) for k in fin), OrderedDict((k, float(r32[k])) for k in fin), fin)


def same_bits(a, b, what):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    assert a.shape == b.shape and np.array_equal(a.view(np.int32), b.view(np.int32)), what


def same_values(a, b, what):
    """bit-exact up to the NaN payload (torch's CPU NaN is not the device's)"""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    assert a.shape == b.shape and np.array_equal(a, b, equal_nan=True), what


# ----------------------------------------------------------------------------------------------------------------
# regimes
# ----------------------------------------------------------------------------------------------------------------
def offset_regime(name):
    """'off+1e4' -> (+1, 1e4)"""
    return (1.0 if name[3] == '+' else -1.0), float(name[4:])


OFFSETS = ['off+1e2', 'off-1e2', 'off+1e4', 'off-1e4', 'off+1e5', 'off-1e5', 'off+1e6', 'off-1e6']
SPECIAL = ['const', 'const_outlier', 'two_valued', 'tiny', 'subnormal', 'huge', 'max']
NONFINITE = ['inf', 'nan', 'inf_pm']
RAW = ['centred'] + OFFSETS + SPECIAL + NONFINITE


def ratio64(x):
    """|mean| / population sd of the finite float64 copy of x"""
    x = np.asarray(x, np.float64).reshape(-1)
    sd = x.std()
    return abs(x.mean()) / sd if sd > 0 else math.inf


def raw_batch(regime, n, seed):
    """n fp32 values of one regime (a torch CPU tensor)"""
    g = cases._g(seed)
    z = torch.randn(n, generator=g, dtype=torch.float64)
    if regime == 'centred':
        x = z
    elif regime.startswith('off'):
        sign, r = offset_regime(regime)
        s = 0.37 if sign > 0 else 3.1  # sd >= 12 fp32 ulps of the mean at 1e6
        x = sign * r * s + s * z
    elif regime == 'const':
        x = torch.full((n, ), 0.1, dtype=torch.float64)  # 0.1f: its square does not sum exactly in a double
    elif regime == 'const_outlier':
        x = torch.full((n, ), 123.456, dtype=torch.float64)
        x[int(torch.randint(0, n, (1, ), generator=g))] = 1123.456
    elif regime == 'two_valued':
        x = torch.where(torch.rand(n, generator=g, dtype=torch.float64) < 0.3, 4096.0, 4096.5)
    elif regime == 'tiny':  # x^2 underflows in fp32
        x = 1e-30 * (3.0 + z)
    elif regime == 'subnormal':
        x = 1e-40 * (3.0 + z)
    elif regime == 'huge':  # x^2 overflows in fp32, the variance does not
        x = 3e19 * (1.0 + 0.1 * z)
    elif regime == 'max':  # near fp32's largest value: the std is representable, the variance is not
        x = 3e38 * (1.0 + 1e-3 * z.clamp(-4.0, 4.0))
    elif regime in NONFINITE:
        x = z.clone()
        i = 1 + torch.randperm(max(n - 1, 1), generator=g)[:2] if n > 2 else torch.tensor([n - 1, n - 1])
        x[i[0]] = math.nan if regime == 'nan' else math.inf
        if regime == 'inf_pm':
            x[i[1]] = -math.inf
    else:
        raise KeyError(regime)
    return x.float()


def check_raw_ratio(regime, x):
    """the ratio a raw batch reached (printed; asserted for the offset regimes)"""
    r = ratio64(x.double().numpy())
    if regime.startswith('off') and x.numel() >= 1000:
        want = offset_regime(regime)[1]
        assert 0.5 * want <= r <= 2.0 * want, (regime, r)
        s = float(x.double().std())
        assert s >= 10 * float(np.spacing(np.float32(abs(float(x.double().mean()))))), (regime, 'sd below 10 ulps')
    return r


def gae_batch(regime, shape, seed, std=None, s=None):
    """gae_data operands of one regime, fp32 CPU tensors: (value, next_value, reward, done, traj_flag, gamma).

    Offset regimes and 'centred': value = next_value = c, done = 0, and a reward that holds the advantage at A + noise:
    r_t = A (1 - f) + (1 - gamma) c + s randn for t < T-1, r_{T-1} = A + (1 - gamma) c + s randn (f = gamma lambda).
    Advantage and return then sit near A and c + A, A = +-ratio * (the advantage's sd, ~ s / sqrt(1 - f^2)), c = A / 2.
    'voff' regimes: the same with A = 0 and c = +-ratio * (the advantage's sd): the offset is in the value alone.
    Special and non-finite regimes: gamma = 0 and value = 0, so that adv = return = reward = the raw batch -- except 'inf' /
    'nan' / 'inf_pm', which keep the gamma > 0 recurrence (a 0 factor would turn an inf into NaN across the step)."""
    g = cases._g(seed)
    T = shape[0]
    B = shape[1] if len(shape) == 2 else 1
    f = GAMMA * LAMBDA
    if regime in SPECIAL:
        r = raw_batch(regime, T * B, seed).reshape(shape)
        z = torch.zeros(shape)
        return z, z.clone(), r, z.clone(), None, 0.0
    voff = regime.startswith('voff')
    sign, ratio = offset_regime(regime[voff:]) if regime[voff:].startswith('off') else (1.0, 0.0)
    s = s or (0.37 if sign > 0 else 3.1)
    A = sign * ratio * s * (ADV_SPREAD if T > 1 else 1.0)  # one step: the advantage is A + s randn
    c = 0.5 * A
    if voff:
        A, c = 0.0, A
    cd = float(np.float32(np.float32(c / std) * np.float32(std))) if std else c  # the value as the kernel decodes it
    z = torch.randn(T, B, generator=g, dtype=torch.float64)
    rw = A * (1.0 - f) + (1.0 - GAMMA) * cd + s * z
    rw[-1] = A + (1.0 - GAMMA) * cd + s * z[-1]
    if regime in NONFINITE:
        i = int(torch.randint(T // 2, T, (1, ), generator=g)) if T > 1 else 0
        j = int(torch.randint(0, B, (1, ), generator=g))
        rw[i, j] = math.nan if regime == 'nan' else math.inf
        if regime == 'inf_pm':  # the next column, or an earlier step of the one sequence (+inf meets -inf there: NaN)
            if B > 1:
                rw[i, (j + 1) % B] = -math.inf
            elif i > 0:
                rw[i // 2, j] = -math.inf
    v = torch.full((T, B), c / std if std else c, dtype=torch.float64)
    shp = (T, ) if len(shape) == 1 else (T, B)
    return (v.float().reshape(shp), v.float().reshape(shp), rw.float().reshape(shp), torch.zeros(shp), None, GAMMA)


def check_gae_ratio(regime, adv, ret):
    ra, rr = ratio64(adv), ratio64(ret)
    if regime.startswith('off') and np.asarray(adv).size >= 1000:
        want = offset_regime(regime)[1]
        assert 0.3 * want <= ra <= 3.0 * want and 0.3 * want <= rr <= 3.0 * want, (regime, ra, rr)
    if regime.startswith('voff') and np.asarray(adv).size >= 1000:
        want = offset_regime(regime[1:])[1]
        assert ra < 0.2 and 0.3 * want <= rr <= 3.0 * want, (regime, ra, rr)
    return ra, rr


# ----------------------------------------------------------------------------------------------------------------
# CPU: the reference, the yardstick and the generators
# ----------------------------------------------------------------------------------------------------------------
def test_reference_and_yardstick_agree_on_dyadic_batches():
    """on a batch whose mean, variance and std are exact in fp32 every path must give the same numbers"""
    x = np.array([1.5, 2.5, 3.5, 4.5, 1.5, 2.5, 3.5, 4.5], np.float32)  # mean 3, pop var 1.25, unbiased var 10/7
    for st in (pop_stats64(x), pop_stats32(x)):
        assert float(st['mean']) == 3.0 and float(st['var']) == 1.25 and st['count'] == 8.0
    y = np.array([1.0, 3.0, 1.0, 3.0, 1.0, 3.0, 1.0, 3.0, 2.0], np.float32)  # mean 2, unbiased var 1
    for t in (torch.from_numpy(y), torch.from_numpy(y).double()):
        st = adv_stats_ref(t)
        assert st['mean'] == 2.0 and st['std'] == float(t.new_tensor(1.0) + 1e-8)
    ok = OrderedDict(mean=2.0, std=1.0 + 1e-8)
    assert check_stats('dyadic', ok, ok, ok) == 0.0
    # a float64 value beyond fp32's range must come back as inf, a NaN variance as 0 in the PPO build
    check_stats('overflow', OrderedDict(mean=1.0, var=math.inf), OrderedDict(mean=1.0, var=math.inf),
                OrderedDict(mean=1.0, var=1e70))
    check_stats('nan var', OrderedDict(mean=math.inf, var=0.0), OrderedDict(mean=math.inf, var=0.0),
                OrderedDict(mean=math.inf, var=math.nan), ppo_var_clamp=True)
    with pytest.raises(AssertionError):
        check_stats('bad', OrderedDict(mean=2.0 * (1 + 1e-5), std=1.0), ok, ok)


@pytest.mark.parametrize('regime', RAW)
def test_raw_regimes_reach_their_ratio(regime):
    x = raw_batch(regime, 100000, 11)
    r = check_raw_ratio(regime, x)
    x64 = x.double()
    if regime == 'const':
        assert float(x64.var()) == 0.0
    elif regime in ('tiny', 'subnormal'):
        assert (x.abs() > 0).all() and float((x * x).abs().max()) < 1e-38
    elif regime in ('huge', 'max'):
        assert torch.isfinite(x).all() and not torch.isfinite(x * x).all()
    elif regime in NONFINITE:
        assert not torch.isfinite(x).all() and torch.isfinite(x[0])
    print('\n[fp64] regime %-14s mean/sd %.3g' % (regime, r))


@pytest.mark.parametrize('regime', ['centred'] + OFFSETS + ['voff+1e4', 'voff-1e2', 'inf'])
def test_gae_regimes_reach_their_ratio(regime):
    for std in (None, VN_STD, 100.0, 0.01):
        v, nv, r, d, tf, gamma = gae_batch(regime, (64, 256), 12, std)
        adv, _, _, unnorm, _ = rl_oracle.ppo_policy_gae_returns(v, nv, r, d, tf, gamma, LAMBDA, std)
        if regime == 'inf':
            assert torch.isinf(adv).any() and torch.isfinite(adv[0, 1:]).any()
            continue
        ra, rr = check_gae_ratio(regime, adv.numpy(), unnorm.numpy())
        print('\n[fp64] gae regime %-10s std %s  adv mean/sd %.3g  return mean/sd %.3g' % (regime, std, ra, rr))


# ----------------------------------------------------------------------------------------------------------------
# GPU: adv_stats_kernel (normalize_advantage; ppo_error_adv_norm without adv_stats)
# ----------------------------------------------------------------------------------------------------------------
# one CTA, 2 CTAs, the 528-CTA cap exactly and one element past it, the grid-stride loop repeating
ADV_SIZES = [1, 2, 2048, 2049, 1081344, 1081345, 4000000]


def _repeat(run, n_runs, multi):
    """run() n_runs times (once for a one-CTA launch); every repeat must give the first run's bits"""
    first = run()
    for _ in range(n_runs - 1 if multi else 0):
        again = run()
        for a, b in zip(first, again):
            same_bits(a, b, 'repeat')
    return first


@pytest.mark.gpu
@pytest.mark.parametrize('n', ADV_SIZES)
@pytest.mark.parametrize('regime', RAW)
def test_adv_stats_fp64(regime, n):
    x = raw_batch(regime, n, 100 + n % 997)
    r = check_raw_ratio(regime, x)
    xd = x.to(DEV)
    norm = b2.normalize_advantage  # (adv - adv.mean()) / (adv.std() + 1e-8), statistics from adv_stats_kernel

    def run():
        st = ops.adv_stats_(xd)
        return st.cpu().numpy(), norm(xd).cpu().numpy()

    st, out = _repeat(run, 3, n > 2048)
    got = OrderedDict(mean=st[0], std=st[1])
    r64 = adv_stats_ref(x.double())
    r32 = adv_stats_ref(xd)
    if n == 1:  # torch.std of one element is NaN
        assert math.isnan(st[1]) and st[0] == x[0].item() or not math.isfinite(x[0].item())
    tag = 'adv_stats %s n=%d (mean/sd %.3g)' % (regime, n, r)
    check_stats(tag, got, r32, r64)
    if regime == 'const' and n > 1:
        assert st[1] == np.float32(1e-8) and st[0] == x[0].item(), (tag, st)
    # the normalised tensor, elementwise, against the float64 normalisation.  Yardstick: the fp32 normalisation with the
    # float64 statistics rounded to fp32 -- fp32 cannot hold the mean closer than half an ulp, and near fp32's largest value
    # torch's fp32 mean / std overflow
    x64 = x.double()
    m64, d64 = x64.mean(), x64.std() + 1e-8
    n64 = ((x64 - m64) / d64).numpy()
    n32 = ((x - m64.float()) / d64.float()).numpy()
    if n > 1:
        compare64(tag + ' normalised', OrderedDict(norm=out), OrderedDict(norm=n32), OrderedDict(norm=n64))


# ----------------------------------------------------------------------------------------------------------------
# GPU: gae_returns -- gae_seq_kernel (1-D, T <= 24576: one CTA) and gae_scan + returns_kernel (longer 1-D, (T, B))
# ----------------------------------------------------------------------------------------------------------------
RET_SHAPES = [
    (1, ), (2, ), (1024, ), (3200, ), (24576, ),  # one CTA
    (24577, ), (100000, ),  # scan + returns_kernel: scalar path, float4 path
    (33, 36), (128, 4096),  # float4 path: 1 and 256 CTAs (config P)
    (67, 1001),  # scalar path, 66 CTAs
    (528, 4096), (529, 4096),  # the float4 cap of 1056 CTAs exactly, and past it
    (1, 1081343), (1, 1081345),  # odd sizes just below and above the scalar cap of 1056 CTAs
]
RET_SPECIAL_SHAPES = [(3200, ), (24577, ), (128, 4096), (1, 1081345)]
RET_OFFSETS = ['centred', 'off+1e2', 'off-1e4', 'off+1e5', 'off-1e6']
# value_norm scales far from 1 on both launch paths: the return statistics must be taken around element 0's return as the
# kernel decodes and encodes it, not around the stored value scaled once more
RET_VN_SHAPES = [(3200, ), (24576, ), (24577, ), (128, 4096)]
VOFFS = ['voff+1e4', 'voff-1e2']
RET_CASES = ([(s, r, std) for s in RET_SHAPES for r in RET_OFFSETS for std in (None, VN_STD)] +
             [(s, r, None) for s in RET_SPECIAL_SHAPES for r in SPECIAL + NONFINITE] +
             [(s, r, VN_STD) for s in RET_SPECIAL_SHAPES for r in ('const', 'nan')] +
             [(s, r, std) for s in RET_VN_SHAPES for r in VOFFS for std in (None, VN_STD)] +
             [(s, r, std) for s in RET_VN_SHAPES for r in ['off-1e4'] + VOFFS for std in (100.0, 0.01)])


def _std_id(std):
    return 'raw' if std is None else ('vn' if std == VN_STD else 'vn%g' % std)


def _multi_cta(shape):
    return not (len(shape) == 1 and shape[0] <= ops.GAE_SEQ_MAX_T)


def _shape_id(s):
    return 'x'.join(map(str, s))


@functools.lru_cache(maxsize=2)
def _ret_oracle(regime, shape, std):
    v, nv, r, d, tf, gamma = gae_batch(regime, shape, 300 + sum(shape) % 1009, std)
    want = rl_oracle.ppo_policy_gae_returns(v.clone(), nv.clone(), r, d, tf, gamma, LAMBDA, std)
    return (v, nv, r, d, tf, gamma), want


@pytest.mark.gpu
@pytest.mark.parametrize('shape,regime,std', RET_CASES,
                         ids=['%s-%s-%s' % (_shape_id(s), r, _std_id(std)) for s, r, std in RET_CASES])
def test_gae_returns_stats_fp64(shape, regime, std):
    (v, nv, r, d, tf, gamma), want = _ret_oracle(regime, shape, std)
    dev = [None if x is None else x.to(DEV) for x in (v, nv, r, d, tf)]

    def run():
        o = b2.gae_returns(b2.gae_data(*dev), gamma, LAMBDA, value_norm_std=std)
        return tuple(t.cpu().numpy() for t in (o.adv, o.value, o.return_, o.unnormalized_return, o.return_stats,
                                               o.adv_stats))

    adv, vout, ret, unnorm, st, ast = _repeat(run, 3, _multi_cta(shape))
    for name, a, b in zip(('adv', 'value', 'return_', 'unnormalized_return'), (adv, vout, ret, unnorm), want[:4]):
        same_values(a, b.numpy(), name)  # pinned by the parity suites: the statistics below describe these tensors
    ra, rr = check_gae_ratio(regime, adv, unnorm)
    tag = 'gae_returns %s %s std=%s (adv mean/sd %.3g, return %.3g)' % (_shape_id(shape), regime, std, ra, rr)
    check_stats(tag + ' return_stats', OrderedDict(mean=st[0], var=st[1], count=st[2]), pop_stats32(unnorm),
                pop_stats64(unnorm), ppo_var_clamp=True)
    if adv.size > 1:
        a32 = torch.from_numpy(adv).to(DEV)
        check_stats(tag + ' adv_stats', OrderedDict(mean=ast[0], std=ast[1]), adv_stats_ref(a32),
                    adv_stats_ref(torch.from_numpy(adv).double()))
    if regime == 'const':
        assert st[1] == 0.0 and ast[1] == np.float32(1e-8), (tag, st, ast)


# ----------------------------------------------------------------------------------------------------------------
# GPU: ppof_gae_returns, all four value_norm modes.  value = next_value = 0 (every mode decodes 0 to 0, PopArt with mu = 0,
# sigma = 1 leaves the reward as it is), so adv is rl_oracle.gae of the reward in every mode.
# ----------------------------------------------------------------------------------------------------------------
PPOF_SHAPES = [(400, ), (24576, ), (24577, ), (128, 4096)]
PPOF_REGIMES = ['centred', 'off+1e4', 'off-1e6', 'const', 'huge', 'nan']


@pytest.mark.gpu
@pytest.mark.parametrize('regime', PPOF_REGIMES)
@pytest.mark.parametrize('shape', PPOF_SHAPES, ids=_shape_id)
@pytest.mark.parametrize('mode', list(ops.VALUE_NORMS))
def test_ppof_gae_returns_stats_fp64(mode, shape, regime):
    _, _, r, d, tf, gamma = gae_batch(regime, shape, 500 + sum(shape) % 1009)
    z = torch.zeros_like(r)
    adv_want = rl_oracle.gae(z.clone(), z.clone(), r, d, tf, gamma, LAMBDA)
    kw = dict(std=VN_STD) if mode == 'baseline' else {}
    if mode == 'popart':
        kw = dict(popart_mu=torch.zeros(1, device=DEV), popart_sigma=torch.ones(1, device=DEV))
    dev = [None if x is None else x.to(DEV) for x in (z, z, r, d, tf)]

    def run():
        o = b2.ppof_gae_returns(b2.gae_data(*dev), gamma, LAMBDA, value_norm=mode, **kw)
        st = o.return_stats.cpu().numpy() if mode == 'baseline' else np.zeros(3, np.float32)
        return o.adv.cpu().numpy(), o.return_.cpu().numpy(), st, o.adv_stats.cpu().numpy()

    adv, ret, st, ast = _repeat(run, 3, _multi_cta(shape))
    same_values(adv, adv_want.numpy(), 'adv')
    tag = 'ppof %s %s %s (adv mean/sd %.3g)' % (mode, _shape_id(shape), regime, ratio64(adv))
    if mode == 'baseline':
        ret_want = adv_want.clone()
        ret_want /= VN_STD  # ppof.py:207: unnormalized_returns /= std, value = 0
        same_values(ret, ret_want.numpy(), 'return_')
        check_stats(tag + ' return_stats', OrderedDict(mean=st[0], var=st[1], count=st[2]), pop_stats32(ret),
                    pop_stats64(ret))  # PPOF's modes keep a NaN variance
    a32 = torch.from_numpy(adv).to(DEV)
    check_stats(tag + ' adv_stats', OrderedDict(mean=ast[0], std=ast[1]), adv_stats_ref(a32),
                adv_stats_ref(torch.from_numpy(adv).double()))
    if regime == 'const':
        assert ast[1] == np.float32(1e-8) and (mode != 'baseline' or st[1] == 0.0), (tag, st, ast)


@pytest.mark.gpu
@pytest.mark.parametrize('std', [VN_STD, 100.0, 0.01], ids=lambda s: 'std%g' % s)
@pytest.mark.parametrize('regime', ['off-1e4'] + VOFFS)
@pytest.mark.parametrize('shape', RET_VN_SHAPES, ids=_shape_id)
def test_ppof_baseline_value_stats_fp64(shape, regime, std):
    """'baseline' with the critic's prediction away from 0: value * std decoded, (value + adv) / std stored and described"""
    pred, npred, r, d, tf, gamma = gae_batch(regime, shape, 600 + sum(shape) % 1009, std)
    value, next_value = pred * std, npred * std  # ppof.py:187-189
    adv_want = rl_oracle.gae(value, next_value, r, d, tf, gamma, LAMBDA)
    ret_want = value + adv_want  # ppof.py:195
    ret_want /= std  # ppof.py:207
    dev = [None if x is None else x.to(DEV) for x in (pred, npred, r, d, tf)]

    def run():
        o = b2.ppof_gae_returns(b2.gae_data(*dev), gamma, LAMBDA, value_norm='baseline', std=std)
        return o.adv.cpu().numpy(), o.return_.cpu().numpy(), o.return_stats.cpu().numpy(), o.adv_stats.cpu().numpy()

    adv, ret, st, ast = _repeat(run, 3, _multi_cta(shape))
    same_values(adv, adv_want.numpy(), 'adv')
    same_values(ret, ret_want.numpy(), 'return_')
    ra, rr = check_gae_ratio(regime, adv, ret)
    tag = 'ppof baseline %s %s std=%g (adv mean/sd %.3g, return %.3g)' % (_shape_id(shape), regime, std, ra, rr)
    check_stats(tag + ' return_stats', OrderedDict(mean=st[0], var=st[1], count=st[2]), pop_stats32(ret),
                pop_stats64(ret))
    check_stats(tag + ' adv_stats', OrderedDict(mean=ast[0], std=ast[1]), adv_stats_ref(torch.from_numpy(adv).to(DEV)),
                adv_stats_ref(torch.from_numpy(adv).double()))


# ----------------------------------------------------------------------------------------------------------------
# GPU: ppo_error_adv_norm end to end on offset-heavy advantages -- statistics from adv_stats_kernel, or from gae_returns
# (config P's composition) -- against float64 normalisation + rl_oracle.ppo_error in float64
# ----------------------------------------------------------------------------------------------------------------
E2E_ADV = {'5+1e-3': (5.0, 1e-3), '-300+0.05': (-300.0, 0.05)}
E2E_SIZES = [(4099, 6), (524288, 6), (4099, 40)]  # tile path; tile path at config P's size; fallback path


def _e2e_runner(p, adv_stats):
    base = _adv_norm_runner(p, DEV)
    if adv_stats is None:
        return base

    def run(t):
        tt = cases.prepare('ppo', t, DEV)
        data = b2.ppo_data(*[tt[k] for k in ('logit_new', 'logit_old', 'action', 'value_new', 'value_old', 'adv',
                                             'return_', 'weight', 'logit_pretrained')])
        loss, info = b2.ppo_error_adv_norm(data, adv_stats=adv_stats, **p)
        res = OrderedDict(('out_' + k, cases._np(v)) for k, v in zip(('policy_loss', 'value_loss', 'entropy_loss',
                                                                      'kl_div'), loss))
        res['out_approx_kl'], res['out_clipfrac'] = np.float32(info.approx_kl), np.float32(info.clipfrac)
        cases._backward('ppo', list(loss), tt, res)
        return res
    return run


@pytest.mark.gpu
@pytest.mark.parametrize('source', ['inside', 'gae_returns'])
@pytest.mark.parametrize('S,N', E2E_SIZES)
@pytest.mark.parametrize('advk', list(E2E_ADV))
def test_ppo_error_adv_norm_offset_fp64(advk, S, N, source):
    m, s = E2E_ADV[advk]
    op, t, p, meta = gen_ppo(7400 + N + S % 97, S, N, clip_ratio=0.2, dual_clip=3.0)
    adv_stats = None
    if source == 'inside':
        g = cases._g(7500 + S % 89)
        t['adv'] = (m + s * torch.randn(S, generator=g, dtype=torch.float64)).float()
    else:  # the advantage gae_returns writes, near m with a spread near s, and its adv_stats
        shape = (128, S // 128) if S % 128 == 0 else (S, )
        regime = 'off%s%r' % ('+' if m > 0 else '-', abs(m) / s)
        v, nv, r, d, tf, gamma = gae_batch(regime, shape, 7600 + S % 83, s=s / ADV_SPREAD)
        o = b2.gae_returns(b2.gae_data(*[None if x is None else x.to(DEV) for x in (v, nv, r, d, tf)]), gamma, LAMBDA)
        want = rl_oracle.ppo_policy_gae_returns(v.clone(), nv.clone(), r, d, tf, gamma, LAMBDA)
        same_bits(o.adv.cpu().numpy(), want[0].numpy(), 'adv')
        t['adv'] = want[0].reshape(-1)
        adv_stats = o.adv_stats
    a64 = t['adv'].double()
    adv64 = rl_oracle.normalize_advantage(a64).numpy()
    frac, bnd, scales = ppo_meta(op, t, p, meta, adv=adv64)
    mix = mixes(op)[0]
    r32, r64 = refs(op, t, p, mix, _adv_norm_runner(p, 'cpu'))
    run = _e2e_runner(p, adv_stats)
    run(t)  # the backward records the mix as the expectation of the next forward
    got = run(t)
    for _ in range(2):
        again = run(t)
        for k in got:
            same_bits(again[k], got[k], 'repeat ' + k)
    tag = 'ppo_error_adv_norm %s S=%d N=%d %s (adv mean/sd %.3g)' % (advk, S, N, source, ratio64(a64.numpy()))
    compare64(tag, got, r32, r64, scales=scales, bnd=bnd, S=S)
    print('[fp64] branches %s %s' % (tag, {k: round(float(v), 3) for k, v in frac.items()}))
