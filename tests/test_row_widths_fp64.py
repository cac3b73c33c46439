"""Every row-width specialisation of the tile kernels against a float64 reference, each case pinned to the kernel it reaches.

Five kernel families take a compile-time row width through ``with_nc`` (csrc/common.cuh): N in WIDTHS gets its own fully
unrolled kernel, every other N the generic one (NC = 0).  Widths divisible by 4 take the float4 branch of
``load_row`` / ``store_row`` (ppo_math.cuh), the other even widths the float2 branch, and the stage layout (and with it
the PPO ring depth) depends on N, ``logit_pretrained`` and ``weight``.

* ``test_instantiation_table`` (no GPU) lists the device kernels of the five families in the built library with
  ``cuobjdump -symbols`` and compares them with TABLE below: a width added to or removed from ``with_nc`` without a table
  entry fails it.  Instantiations that no accepted input reaches are listed in UNREACHABLE with the host predicate that
  rules them out.
* The GPU sweep runs every reachable entry, and the generic kernel at widths either side of a table width, on the
  adversarial generators of test_offpolicy_fp64 (both masks, dual clip, the operand sets that change the stage layout),
  through the forward-written gradients, the verify launch's recompute and the separate backward, and compares with the
  float64 reference under the same bound K.  Each case runs once more under torch.profiler and asserts the launched
  kernels of these families are exactly the ones its table entries name.
"""
import ctypes
import os
import re
import shutil
import subprocess
from collections import OrderedDict

import pytest
import torch

from di_engine_b200 import _lib, ops
from oracle import rl_oracle
from tests import cases
from tests.test_offpolicy_fp64 import (DEV, MASKS, VT_PARAMS, _Mix, _run_gae_ppo, check_branches, compare64, gen_ppo,
                                       gen_vtrace, gpu_paths, mixes, ppo_meta, refs, ring_wrap_rows, run_gpu_api,
                                       vtrace_scales, zero_at_masked)

WIDTHS = (2, 3, 4, 5, 6, 7, 8, 9, 10, 12, 14, 16, 18)  # with_nc's compile-time widths
GENERIC = (11, 19)  # the generic kernel (NC = 0): just above 10 / below 12, and just above the widest table width
PS_R = 256  # rows per stage of ppo_tile_kernel (ppo.cu PS_R)
PS_MAX_STAGES = 8
PS_SMEM_LIMIT = 227 * 1024 - 1024
ROWS_RPT2 = 256 * 132 * 4  # fused.cu dispatch_fused: two rows per thread from four 256-row tiles per SM (NUM_SMS = 132)

# ----------------------------------------------------------------------------------------------------------------
# the instantiation table: (family, template arguments after NC) -> what reaches it, for every NC in (0,) + WIDTHS
# ----------------------------------------------------------------------------------------------------------------
TABLE = OrderedDict([
    (('ppo_tile_kernel', (0, )), ('ppo_error / ppo_policy_error / happo_error, G == 1, N <= 32, 16-byte aligned, '
                                  'ops.PPO_FUSED_BACKWARD = False: the forward launch (FWD)', 'ppo:wrap S = ring wrap')),
    (('ppo_tile_kernel', (1, )), ('the same with the fused backward: the forward launch writes the gradients '
                                  '(FWD_GRAD)', 'ppo:wrap / ppo:pre / ppo:happo, S = 4099')),
    (('ppo_tile_kernel', (2, )), ('the backward launch (BWD): the one-stage verify launch after FWD_GRAD or after '
                                  'gae_ppo_error, the full ring after FWD', 'ppo:wrap')),
    (('gae_ppo_kernel', (1, 1)), ('gae_ppo_error, b200rl_gae_ppo_set_impl(1), T * B < %d' % ROWS_RPT2,
                                  'gae:small T, B = 33, 20')),
    (('gae_ppo_kernel', (0, 1)), ('the same, inputs without requires_grad', 'gae:small')),
    (('gae_ppo_kernel', (1, 2)), ('gae_ppo_error, set_impl(1), T * B >= %d: two rows per thread' % ROWS_RPT2,
                                  'gae:rpt2 T, B = 136, 1000')),
    (('gae_ppo_kernel', (0, 2)), ('the same, inputs without requires_grad', 'gae:rpt2')),
    (('gae_ppo_ws_kernel', (1, 16)), ('gae_ppo_error, b200rl_gae_ppo_set_impl(2), B far below 32 per SM',
                                      'gae:small')),
    (('gae_ppo_ws_kernel', (0, 16)), ('the same, inputs without requires_grad', 'gae:small')),
    (('gae_ppo_ws_kernel', (1, 32)), ('gae_ppo_error, set_impl(2), about 32 columns per SM (cw_pick_tc, the '
                                      'device SM count)', 'gae:wide T, B = 9, 32 * SMs')),
    (('gae_ppo_ws_kernel', (0, 32)), ('the same, inputs without requires_grad', 'gae:wide')),
    (('vt_rows_tile_kernel', ()), ('vtrace_error_discrete_action, ops.VTRACE_FUSED = False, N <= 32: forward rows',
                                   'vt:small T, B = 33, 20')),
    (('vt_bwd_tile_kernel', ()), ('the same: backward rows', 'vt:small')),
    (('vtrace_ws_kernel', (1, 16)), ('vtrace_error_discrete_action, set_impl(0), vtws_ok, B <= 4224 (2 * 132 '
                                     '16-column tiles)', 'vt:small')),
    (('vtrace_ws_kernel', (0, 16)), ('the same, inputs without requires_grad', 'vt:small')),
    (('vtrace_ws_kernel', (1, 32)), ('set_impl(0), vtws_ok, B > 4224', 'vt:wide T, B = 5, 4352')),
    (('vtrace_ws_kernel', (0, 32)), ('the same, inputs without requires_grad', 'vt:wide')),
    (('vtrace_res_kernel', (1, 4)), ('set_impl(2) (or set_impl(0) where vtws_ok fails), B % 8 != 0', 'vt:small')),
    (('vtrace_res_kernel', (0, 4)), ('the same, inputs without requires_grad', 'vt:small')),
    (('vtrace_res_kernel', (1, 8)), ('set_impl(2) (or set_impl(0) where vtws_ok fails), B % 8 == 0',
                                     'vt:res8 T, B = 24, 64')),
    (('vtrace_res_kernel', (0, 8)), ('the same, inputs without requires_grad', 'vt:res8')),
])
FAMILIES = sorted({f for f, _ in TABLE})

# instantiated, but no accepted input reaches them: vtws_ok (vtws.cu) needs vw_pick_stages(N, has_weight) >= 3, three
# 32-column stages in 112 KB, which holds for N <= 15 only; wider rows go to the resident kernel (or are refused)
UNREACHABLE = {('vtrace_ws_kernel', (nc, grads, tc)): 'vtws_ok: vw_pick_stages(%d, w) < 3' % nc
               for nc in (16, 18) for grads in (0, 1) for tc in (16, 32)}


def table_entries():
    return {(f, (nc, ) + rest) for f, rest in TABLE for nc in (0, ) + WIDTHS}


def nc_of(N):
    return N if N in WIDTHS else 0


def vtws_fits(N, has_w=True):
    """vtws.cu vw_pick_stages(N, has_w) >= 3 (with its default 32-column rows): the streaming V-trace kernel takes N"""
    ct, row = 256, 32 * 4
    stage = ct * (2 * N * 4 + 8 + (4 if has_w else 0)) + (ct * 4 + row) + ct * 4 + ct * 4 + (ct * 4 + row)
    return N <= 32 and 3 * stage + 4 * 4 * 8 + 64 <= 112 * 1024


# ----------------------------------------------------------------------------------------------------------------
# kernel names: cuobjdump symbols (mangled) and profiler events (demangled) -> (family, template arguments)
# ----------------------------------------------------------------------------------------------------------------
_NAME = re.compile(r'(?:^|[\s:])(%s)<([^<>]*)>\(' % '|'.join(FAMILIES))


def _arg(s):
    s = re.sub(r'^\((?:int|bool)\)', '', s.strip())
    return {'true': 1, 'false': 0}.get(s, None) if not s.lstrip('-').isdigit() else int(s)


def entry_of(demangled):
    m = _NAME.search(demangled)
    if not m:
        return None
    return m.group(1), tuple(_arg(x) for x in m.group(2).split(','))


def _tool(name):
    for d in (os.environ.get('CUDA_HOME'), '/usr/local/cuda'):
        if d and os.path.isfile(os.path.join(d, 'bin', name)):
            return os.path.join(d, 'bin', name)
    return shutil.which(name)


def _demangle(names):
    if not names:
        return []
    out = subprocess.run([_tool('cu++filt')], input='\n'.join(names), capture_output=True, text=True, check=True).stdout
    return out.splitlines()


def library_entries():
    """the table families' device kernels in the built library (cuobjdump reads the sm_90a cubins, no GPU needed)"""
    out = subprocess.run([_tool('cuobjdump'), '-symbols', _lib.LIB_PATH], capture_output=True, text=True, check=True)
    mangled = sorted({ln.split()[-1] for ln in out.stdout.splitlines() if 'STO_ENTRY' in ln})
    return {e for e in map(entry_of, _demangle(mangled)) if e}


def test_instantiation_table():
    assert _tool('cuobjdump') and _tool('cu++filt'), 'the CUDA toolkit that built the library: cuobjdump, cu++filt'
    _lib.load()
    got, want = library_entries(), table_entries()
    assert got == want, ('in the library, not in TABLE', sorted(got - want), 'in TABLE, not in the library',
                         sorted(want - got))
    assert set(UNREACHABLE) <= want
    for f, args in UNREACHABLE:  # the predicate holds for exactly these widths
        assert not vtws_fits(args[0])
    assert all(vtws_fits(n) for n in WIDTHS + GENERIC if n < 16)


def test_sweep_cases_cover_every_reachable_entry():
    """the union of what the GPU cases below expect to launch is every table entry but the unreachable ones"""
    expected = set()
    for run, N in all_runs():
        expected |= run_expectations(run, N)
    reachable = table_entries() - set(UNREACHABLE)
    assert expected == reachable, ('not reached', sorted(reachable - expected), 'not in the table',
                                   sorted(expected - reachable))


# ----------------------------------------------------------------------------------------------------------------
# ppo_tile_kernel geometry (host arithmetic, no GPU): every table width and both generic neighbours
# ----------------------------------------------------------------------------------------------------------------
def stage_bytes(N, pre, w):
    """ppo_math.cuh ppo_layout for a 256-row stage, rounded to 128 bytes"""
    b = PS_R * N * 4 * (3 if pre else 2) + PS_R * 8 + 4 * PS_R * 4 + (PS_R * 4 if w else 0)
    return (b + 127) & ~127


def geometry(S, N, pre=False, w=False, verify=False, sms=132):
    g = (ctypes.c_longlong * 3)()
    assert _lib.load().b200rl_ppo_tile_geometry(S, N, int(pre), int(w), int(verify), sms, g) == 0
    return {'grid': g[0], 'stages': g[1], 'smem': g[2]}


@pytest.mark.parametrize('N', WIDTHS + GENERIC)
def test_ppo_tile_geometry_at_every_width(N):
    bars = 2 * PS_MAX_STAGES * 8
    for pre in (False, True):
        for w in (False, True):
            st = stage_bytes(N, pre, w)
            g = geometry(524288, N, pre, w)
            stages = min(PS_MAX_STAGES, (PS_SMEM_LIMIT - bars) // st)
            assert g == {'grid': 132, 'stages': stages, 'smem': stages * st + bars}, (N, pre, w, g, st)
            v = geometry(524288, N, pre, w, verify=True)
            assert v == {'grid': 132, 'stages': 1, 'smem': st + bars}, (N, pre, w, v)
            assert v['smem'] < g['smem'] or stages == 1
            # small batches: no deeper ring than a CTA has tiles; the ragged last tile counts as one
            assert geometry(PS_R * 3 + 1, N, pre, w) == {'grid': 4, 'stages': 1, 'smem': st + bars}
            for sms in (132, 114, 78):
                ring_wrap_rows(N, pre, w, sms)


# ----------------------------------------------------------------------------------------------------------------
# the cases: (run, N) -> the table entries its launches must be, and how it runs
# ----------------------------------------------------------------------------------------------------------------
PPO_RUNS = ('wrap', 'pre', 'happo')
GAE_RUNS = {'small': ((33, 20), ('row', 'col')), 'rpt2': ((136, 1000), ('row', )), 'wide': ((9, 'sms'), ('col', ))}
VT_RUNS = {'small': ((33, 20), ('pg', 'auto', 'resident')), 'wide': ((5, 4352), ('auto', )),
           'res8': ((24, 64), ('resident', ))}


def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132


def gae_shape(size):
    """(T, B) of a gae case; 'wide' takes B = 32 columns per SM, where cw_pick_tc picks 32-column tiles"""
    T, B = GAE_RUNS[size][0]
    return T, (32 * sm_count() if B == 'sms' else B)


def cw_pick_tc(N, has_w, B, sms, has_pre=False):
    """colws.cu cw_pick_tc: 16 or 32 columns per tile on a device with `sms` SMs (the runtime SM count)"""
    raw_arr = 256 * 4
    stage = (256 * ((3 if has_pre else 2) * N * 4 + 8 + 12 + (4 if has_w else 0)) + 127) & ~127

    def stages(tc):
        ms, rs, limit = (8, 4, 227 * 1024) if tc == 32 else (4, 2, 112 * 1024)
        fits = [k for k in range(2, ms + 1) if k * stage + rs * 5 * raw_arr + ms * raw_arr + raw_arr + 3 * ms * 8 + 32 <= limit]
        return max(fits) if fits else 0

    if stages(32) < 2 * stages(16):
        return 16
    n16, n32 = -(-B // 16), -(-B // 32)
    if n32 < sms - sms // 16:
        return 16
    return 32 if 32 * -(-n32 // sms) <= 16 * -(-n16 // sms) else 16


def all_runs():
    for N in WIDTHS + GENERIC:
        for r in PPO_RUNS:
            yield 'ppo:' + r, N
        for r in GAE_RUNS:
            yield 'gae:' + r, N
        for r in VT_RUNS:
            yield 'vt:' + r, N


def launch_expectations(run, N, impl):
    """-> [(label, {entries})]: the launches of one impl of a case, each with the table entries it must launch"""
    nc = nc_of(N)
    kind, size = run.split(':')
    if kind == 'ppo':
        return [('fused', {('ppo_tile_kernel', (nc, 1)), ('ppo_tile_kernel', (nc, 2))}),
                ('separate', {('ppo_tile_kernel', (nc, 0)), ('ppo_tile_kernel', (nc, 2))})]
    if kind == 'gae':
        # the backward of either is ppo.cu's verify launch
        bwd = {('ppo_tile_kernel', (nc, 2))}
        if impl == 'row':
            rpt = 2 if size == 'rpt2' else 1
            return [('grads', {('gae_ppo_kernel', (nc, 1, rpt))} | bwd), ('forward', {('gae_ppo_kernel', (nc, 0, rpt))})]
        tc = cw_pick_tc(N, size != 'wide', gae_shape(size)[1], sm_count())
        return [('grads', {('gae_ppo_ws_kernel', (nc, 1, tc))} | bwd), ('forward', {('gae_ppo_ws_kernel', (nc, 0, tc))})]
    B = VT_RUNS[size][0][1]
    if impl == 'pg':
        return [('grads', {('vt_rows_tile_kernel', (nc, )), ('vt_bwd_tile_kernel', (nc, ))})]
    if impl == 'auto' and vtws_fits(N):
        tc = 32 if (B + 15) // 16 > 2 * 132 else 16  # dispatch_vtws: the compile-time NUM_SMS = 132
        return [(g, {('vtrace_ws_kernel', (nc, gi, tc))}) for g, gi in (('grads', 1), ('forward', 0))]
    tc = 8 if B % 8 == 0 else 4  # vr_pick_tc: the resident tile fits at these short T
    return [(g, {('vtrace_res_kernel', (nc, gi, tc))}) for g, gi in (('grads', 1), ('forward', 0))]


def run_impls(run):
    kind, size = run.split(':')
    if kind == 'ppo':
        return ('tile', )
    return (GAE_RUNS if kind == 'gae' else VT_RUNS)[size][1]


def run_expectations(run, N):
    out = set()
    for impl in run_impls(run):
        for _, e in launch_expectations(run, N, impl):
            out |= e
    return out


# ----------------------------------------------------------------------------------------------------------------
# GPU: launch log and helpers
# ----------------------------------------------------------------------------------------------------------------
LAUNCHED = {}  # entry -> the first case that launched it; every case pins its launches after its float64 comparisons


def launched_names(fn):
    """the demangled names of the kernels one call of fn launches (torch.profiler, CUDA activity)"""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    mangled = [n for n in names if n.startswith('_Z')]
    return [n for n in names if not n.startswith('_Z')] + _demangle(mangled)


def pin(tag, fn, want):
    """The table-family kernels fn launches must be exactly ``want``.  Which kernels a call launches is decided on the host
    from shapes, addresses and options alone, so a trace that shows a kernel outside ``want`` fails at once.  A trace that
    lacks one of ``want`` is one whose activity records were not all delivered: fn is traced again, at most five times,
    and every trace is in the failure message."""
    traces = []
    for _ in range(5):
        names = launched_names(fn)
        got = {e for e in map(entry_of, names) if e}
        traces.append(names)
        assert got <= want, (tag, 'launched', sorted(got), 'table entries', sorted(want), 'trace', names)
        if got == want:
            break
    assert got == want, (tag, 'table entries', sorted(want), 'traces', traces)
    for e in got:
        LAUNCHED.setdefault(e, tag)
    print('[pin] %-40s %s%s' % (tag, ' '.join('%s<%s>' % (f, ','.join(map(str, a))) for f, a in sorted(got)),
                                '' if len(traces) == 1 else '  (%d traces)' % len(traces)))


class _NoGrad:
    """run_api / prepare leave every input without requires_grad: the forward-only kernels (GRADS = false)"""

    def __init__(self, op):
        self.op = op

    def __enter__(self):
        self.old = cases.GRAD_INPUTS[self.op]
        cases.GRAD_INPUTS[self.op] = []

    def __exit__(self, *exc):
        cases.GRAD_INPUTS[self.op] = self.old


def losses_only(r):
    return OrderedDict((k, v) for k, v in r.items() if k.startswith('out_'))


def branches(tag, frac):
    print('[fp64] branches %s %s' % (tag, {k: round(float(v), 3) for k, v in frac.items()}))


def masks_for(N):
    """both masks at every width: the first case of a width takes one, the second the other"""
    return sorted(MASKS)[N % 2], sorted(MASKS)[1 - N % 2]


# ----------------------------------------------------------------------------------------------------------------
# ppo_tile_kernel: FWD, FWD_GRAD and BWD (verify launch and full ring), ring wrap, logit_pretrained, HAPPO's factor
# ----------------------------------------------------------------------------------------------------------------
def ppo_batch(run, N):
    m1, m2 = masks_for(N)
    seed = 8000 + 100 * PPO_RUNS.index(run) + N
    if run == 'wrap':
        S = ring_wrap_rows(N, False, True)  # the device's SM count
        return gen_ppo(seed, S, N, mask=m1, weight=True, clip_ratio=0.2, dual_clip=3.0), m1
    if run == 'pre':
        kl = ('k1', 'k2', 'k3')[N % 3]
        return gen_ppo(seed, 4099, N, mask=m2, weight=False, pretrained=True, clip_ratio=0.2, dual_clip=3.0,
                       kl_type=kl), m2 + ' ' + kl
    op, t, p, meta = gen_ppo(seed, 4099, N, mask=m2, clip_ratio=0.2, dual_clip=3.0)
    t = OrderedDict((k, t[k]) for k in cases.HAPPO_FIELDS if k != 'factor')
    t['factor'] = torch.rand(4099, 1, generator=cases._g(seed + 50)) * 2.7 + 0.3  # factor * min crosses the floor
    return ('happo', t, p, meta), m2


def check_ppo(run, N):
    (op, t, p, meta), desc = ppo_batch(run, N)
    tag = 'ppo:%s N%d %s S%d' % (run, N, desc, len(t['adv']))
    a, b = mixes(op)
    frac, bnd, scales = ppo_meta(op, t, p, meta)
    check_branches(frac, ['ratio_clipped', 'dual_floor', 'on_policy', 'masked_rows', 'value_clipped'])
    rr = (refs(op, t, p, a), refs(op, t, p, b))
    run_gpu = run_gpu_api(op, t, p)
    try:
        for label, want in launch_expectations('ppo:' + run, N, 'tile'):
            ops.PPO_FUSED_BACKWARD = label == 'fused'
            for path, i, got in gpu_paths(op, run_gpu, a, b):
                compare64('%s %s %s' % (tag, label, path), got, *rr[i], scales=scales, bnd=bnd, S=len(bnd))
                zero_at_masked(tag, got, 'grad_logit_new', meta['masked'].numpy())
            with _Mix(op, a):
                run_gpu()  # the expectation the fused forward writes for
                pin('%s %s' % (tag, label), run_gpu, want)
    finally:
        ops.PPO_FUSED_BACKWARD = True
    branches(tag, frac)


@pytest.mark.gpu
@pytest.mark.parametrize('run', PPO_RUNS)
@pytest.mark.parametrize('N', WIDTHS + GENERIC)
def test_ppo_tile_width_fp64(N, run):
    check_ppo(run, N)


# ----------------------------------------------------------------------------------------------------------------
# gae -> ppo_error in one launch: row tiles (one and two rows per thread) and column tiles (16 and 32 columns)
# ----------------------------------------------------------------------------------------------------------------
def gae_batch(size, N):
    T, B = gae_shape(size)
    mask = masks_for(N)[list(GAE_RUNS).index(size) % 2]
    seed = 8400 + 100 * list(GAE_RUNS).index(size) + N
    _, tg, pg = cases.gae_case(seed, T, B, p_done=0.03, gamma=0.99, lambda_=0.95)
    op, tp, p, meta = gen_ppo(seed + 50, T * B, N, mask=mask, weight=size != 'wide', clip_ratio=0.2, dual_clip=3.0)
    og = {k: v.clone() for k, v in tg.items()}
    adv = rl_oracle.gae(og['value'], og['next_value'], og['reward'], og['done'], og['traj_flag'], **pg)
    tp['adv'] = adv.reshape(-1)  # the fp32 advantage feeds both references: the kernel must reproduce it bit for bit
    return tg, pg, og['next_value'], adv, tp, p, meta, mask


def check_gae(size, N):
    tg, pg, nv, adv, tp, p, meta, mask = gae_batch(size, N)
    tag = 'gae:%s N%d %s %dx%d' % (size, N, mask, *gae_shape(size))
    a, b = mixes('ppo')
    frac, bnd, scales = ppo_meta('ppo', tp, p, meta)
    check_branches(frac, ['ratio_clipped', 'dual_floor', 'on_policy', 'masked_rows', 'value_clipped'])
    rr = (refs('ppo', tp, p, a), refs('ppo', tp, p, b))
    run_gpu = lambda: _run_gae_ppo(tg, pg, tp, p, nv, adv)  # noqa: E731  asserts adv and next_value bit for bit

    def run_fwd():
        with _NoGrad('ppo'):
            return run_gpu()

    for impl in GAE_RUNS[size][1]:
        old = ops.lib().b200rl_gae_ppo_set_impl({'row': 1, 'col': 2}[impl])
        try:
            for path, i, got in gpu_paths('ppo', run_gpu, a, b):
                compare64('%s %s %s' % (tag, impl, path), got, *rr[i], scales=scales, bnd=bnd, S=len(bnd))
                zero_at_masked(tag, got, 'grad_logit_new', meta['masked'].numpy())
            with _Mix('ppo', a):
                compare64('%s %s forward only' % (tag, impl), run_fwd(), *map(losses_only, rr[0]), scales=scales,
                          bnd=bnd, S=len(bnd))
            for label, want in launch_expectations('gae:' + size, N, impl):
                with _Mix('ppo', a):
                    pin('%s %s %s' % (tag, impl, label), run_gpu if label == 'grads' else run_fwd, want)
        finally:
            ops.lib().b200rl_gae_ppo_set_impl(old)
    branches(tag, frac)


@pytest.mark.gpu
@pytest.mark.parametrize('size', list(GAE_RUNS))
@pytest.mark.parametrize('N', WIDTHS + GENERIC)
def test_gae_ppo_width_fp64(N, size):
    check_gae(size, N)


# ----------------------------------------------------------------------------------------------------------------
# V-trace: pg.cu row tiles, vtws.cu streaming column tiles (16 / 32 columns) and resident tiles (4 / 8 columns)
# ----------------------------------------------------------------------------------------------------------------
VT_IMPL = {'auto': 0, 'resident': 2, 'pg': 0}


def vtrace_value_scale(t, p):
    """Scale of the V-trace value loss L for the bound: L plus the spread of its first-order response to fp32 rounding of
    each row's log-sum-exp.  An fp32 log-sum-exp is rounded at the magnitude of the row's largest logit (the generator
    shifts rows by up to 50, where one ulp is 2^-18), and that rounding moves log pi(a) and with it the importance weight
    of every transition; the scan carries the change into vs at every earlier step.  With independent roundings of
    2^-24 * |max z| per row the first-order change of L has standard deviation
        2^-24 * sqrt(sum_i (dL/d log isw_i * (|max z_target,i| + |max z_behaviour,i|))^2),
    computed here in float64.  The scale returned is L plus that root sum of squares (compare64's floor is 2^-24 times
    it).  The fp32 oracle makes the same roundings, so its own error is one draw of the same quantity and can be far below
    it by chance."""
    zt, zb, act = t['target_output'].double(), t['behaviour_output'].double(), t['action']
    lt = torch.log_softmax(zt, -1).gather(-1, act[..., None])[..., 0]
    lb = torch.log_softmax(zb, -1).gather(-1, act[..., None])[..., 0]
    log_isw = (lt - lb).requires_grad_(True)
    isw = log_isw.exp()
    v, r, w = t['value'].double(), t['reward'].double(), t['weight'].double()
    rho, cs = isw.clamp(max=p['rho_clip_ratio']), isw.clamp(max=p['c_clip_ratio'])
    deltas = rho * (r + p['gamma'] * v[1:] - v[:-1])
    carry, vs = torch.zeros_like(r[0]), []
    for i in range(r.shape[0] - 1, -1, -1):
        carry = deltas[i] + p['gamma'] * p['lambda_'] * cs[i] * carry
        vs.append(v[i] + carry)
    loss = ((v[:-1] - torch.stack(vs[::-1])) ** 2 * w).mean()
    loss.backward()
    mag = zt.amax(-1).abs() + zb.amax(-1).abs()  # the row maxima: never masked (the chosen action is not)
    return float(loss.detach()) + float((log_isw.grad * mag).pow(2).sum().sqrt())


def check_vtrace(size, N):
    (T, B), impls = VT_RUNS[size]
    mask = masks_for(N)[list(VT_RUNS).index(size) % 2]
    op, t, p, meta = gen_vtrace(8700 + 100 * list(VT_RUNS).index(size) + N, T, B, N, mask=mask, **VT_PARAMS)
    tag = 'vt:%s N%d %s %dx%d' % (size, N, mask, T, B)
    a, b = mixes(op)
    scales, frac = vtrace_scales(t, p)
    scales['out_value_loss'] = vtrace_value_scale(t, p)
    frac['on_policy'] = float(meta['on'].double().mean())
    frac['masked_rows'] = float(meta['masked'].any(-1).double().mean())
    check_branches(frac, ['is_far_above', 'is_far_below', 'on_policy', 'masked_rows'])
    rr = (refs(op, t, p, a), refs(op, t, p, b))
    run_gpu = run_gpu_api(op, t, p)

    def run_fwd():
        with _NoGrad(op):
            return run_gpu()

    for impl in impls:
        old = ops.lib().b200rl_vtrace_set_impl(VT_IMPL[impl])
        ops.VTRACE_FUSED = impl != 'pg'
        try:
            for path, i, got in gpu_paths(op, run_gpu, a, b):
                compare64('%s %s %s' % (tag, impl, path), got, *rr[i], scales=scales)
                zero_at_masked(tag, got, 'grad_target_output', meta['masked'].numpy())
            if impl != 'pg':
                with _Mix(op, a):
                    compare64('%s %s forward only' % (tag, impl), run_fwd(), *map(losses_only, rr[0]), scales=scales)
            for label, want in launch_expectations('vt:' + size, N, impl):
                with _Mix(op, a):
                    pin('%s %s %s' % (tag, impl, label), run_gpu if label == 'grads' else run_fwd, want)
        finally:
            ops.VTRACE_FUSED = True
            ops.lib().b200rl_vtrace_set_impl(old)
            ops.vtrace_hint(torch.device(DEV)).copy_(torch.tensor(cases.LOSS_MIX['vtrace']))
    branches(tag, frac)


@pytest.mark.gpu
@pytest.mark.parametrize('size', list(VT_RUNS))
@pytest.mark.parametrize('N', WIDTHS + GENERIC)
def test_vtrace_width_fp64(N, size):
    check_vtrace(size, N)


# ----------------------------------------------------------------------------------------------------------------
# coverage: every reachable table entry launched by a case whose results passed the float64 comparison (a case that did not
# run in this session, e.g. deselected, runs here in full)
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_every_reachable_entry_compared_and_launched():
    reachable = table_entries() - set(UNREACHABLE)
    check = {'ppo': check_ppo, 'gae': check_gae, 'vt': check_vtrace}
    for run, N in all_runs():
        if not run_expectations(run, N) <= set(LAUNCHED):
            kind, size = run.split(':')
            check[kind](size, N)
    missing = reachable - set(LAUNCHED)
    print('\n[pin] %d of %d reachable table entries compared with float64 and launched; %d unreachable: %s' % (
        len(reachable & set(LAUNCHED)), len(reachable), len(UNREACHABLE), sorted(UNREACHABLE)))
    assert not missing, sorted(missing)
    assert not set(LAUNCHED) - reachable, sorted(set(LAUNCHED) - reachable)
