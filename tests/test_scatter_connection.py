"""ScatterConnection (ding/torch_utils/network/scatter_connection.py:30-121) on csrc/scatter.cu, and the ``hpc_rll`` shim's
``torch_utils`` half (ding/hpc_rl/wrapper.py:62-73: ScatterConnection, LSTM).

CPU (``-m "not gpu"``):
  * with ``install_hpc_rll()`` and ``ding.enable_hpc_rl`` set, the reference's rnn.py imports (it imports
    ``hpc_rll.torch_utils.network.rnn`` at the top) and ``lstm_type='hpc'`` raises NotImplementedError;
  * the live reference ``hpc_wrapper`` dispatches ScatterConnection.forward into the shim for the positional, keyword and
    mixed call forms, reuses the cached instance and reaches ``b200rl_scatter_fwd`` (a recording stand-in for the library);
  * ``install()`` patches forward / xy_forward on the reference class, instances built earlier included, and
    ``uninstall()`` restores them;
  * TypeError for a non-fp32 x or a non-int64 index, IndexError before any launch under ``B200RL_CHECK_INDICES=1``;
  * the fixtures in ``tests/golden/scatter/`` regenerate from their seeds.
GPU: bit-identical to the reference run on the CPU (forward in both modes and d x) on the reference HPC test's shape, the
football map, many entities per cell, M = 0, B = 1, N = 1 / 33 / 257, a 128 x 128 map, wrapped (y, W) indices, strided
views, xy_forward and the reference's unit tests; against the reference on the same CUDA tensors; determinism; guarded
out-of-range entities; the fixtures; torch.compile(fullgraph=True).
"""
import contextlib
import glob
import importlib
import json
import os
import sys

import numpy as np
import pytest
import torch

import di_engine_b200 as b2
from di_engine_b200 import _lib, ops
from di_engine_b200.torch_utils import scatter_connection as sc
from oracle import ref_scatter

HAVE_REF = ref_scatter.available()
GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'scatter')
SAMPLE = 4096  # a fixture stores a larger tensor as a seeded sample of this many entries and its float64 sum
gpu = pytest.mark.gpu
need_ref = pytest.mark.skipif(not HAVE_REF, reason='reference archive not built')


def _case(seed, B, M, N, H, W, form='location', wrap=False):
    return dict(seed=seed, B=B, M=M, N=N, H=H, W=W, form=form, wrap=wrap)


# the reference HPC test's shape (ding/hpc_rl/tests/test_scatter.py:9-13); gfootball's spatial encoder at B = 64
# (football_q_network.py:203,243: 22 players, 32 attributes, 84 x 200); the rest are edges of the tiling
CASES = {
    'hpc': _case(1, 256, 256, 256, 16, 16),
    'football': _case(2, 64, 22, 32, 84, 200),
    'many_per_cell': _case(3, 8, 1024, 64, 4, 4),
    'm0': _case(4, 3, 0, 5, 4, 6),
    'b1': _case(5, 1, 40, 16, 5, 7),
    'n1': _case(6, 4, 30, 1, 6, 6),
    'n33': _case(7, 4, 300, 33, 8, 9),
    'n33_sparse': _case(8, 3, 5, 33, 20, 30),
    'n257': _case(9, 2, 100, 257, 12, 11),
    'map128': _case(10, 4, 512, 16, 128, 128),
    'chunks': _case(11, 2, 1100, 8, 40, 40),
    'wrap': _case(12, 6, 200, 24, 10, 12, wrap=True),
    'xy': _case(13, 10, 20, 3, 13, 17, form='xy'),
    'naive': _case(14, 2, 24, 32, 2, 3),
}
GOLDEN_CASES = ('football_b2', 'hpc_b2', 'many_per_cell_b1', 'naive', 'wrap', 'xy')


def golden_case(name):
    c = dict(CASES[name.rsplit('_b', 1)[0]] if name.endswith(('_b1', '_b2')) else CASES[name])
    if name.endswith(('_b1', '_b2')):
        c['B'] = int(name[-1])
    return c


def make_inputs(c):
    """x (B, M, N) and the index: location (B, M, 2) as (y, x), or (coord_x, coord_y) for xy_forward; ``wrap`` puts a
    quarter of the entities at column W of a row below the last, which is cell (y + 1, 0)"""
    g = torch.Generator().manual_seed(c['seed'])
    B, M, N, H, W = c['B'], c['M'], c['N'], c['H'], c['W']
    x = torch.randn(B, M, N, generator=g)
    if c['form'] == 'xy':
        return x, (torch.randint(0, H, (B, M), generator=g), torch.randint(0, W, (B, M), generator=g))
    h = torch.randint(0, H, (B, M), generator=g)
    w = torch.randint(0, W, (B, M), generator=g)
    if c['wrap']:
        sel = torch.rand(B, M, generator=g) < 0.25
        h = torch.where(sel, torch.randint(0, H - 1, (B, M), generator=g), h)
        w = torch.where(sel, torch.full_like(w, W), w)
    return x, (torch.stack([h, w], dim=2), )


def upstream(c, seed=99):
    return torch.randn(c['B'], c['N'], c['H'], c['W'], generator=torch.Generator().manual_seed(seed))


def run(model, c, x, index, g, device):
    """the map and d x of ``model`` on ``device`` for the upstream gradient g (numpy)"""
    x = x.detach().to(device).clone().requires_grad_(True)
    index = [t.to(device) for t in index]
    if c['form'] == 'xy':
        out = model.xy_forward(x, (c['H'], c['W']), *index)
    else:
        out = model(x, (c['H'], c['W']), *index)
    out.backward(g.to(device))
    return out.detach().cpu().numpy(), x.grad.cpu().numpy()


@contextlib.contextmanager
def reference_cls():
    with ref_scatter.network():
        yield ref_scatter.scatter_connection().ScatterConnection


def sample(a):
    a = np.asarray(a).reshape(-1)
    if a.size <= SAMPLE:
        return a, None
    idx = np.sort(np.random.default_rng(a.size).choice(a.size, SAMPLE, replace=False))
    return a[idx], np.float64(a.astype(np.float64).sum())


def input_sums(x, index):
    return np.array([float(x.double().sum())] + [float(t.double().sum()) for t in index])


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------
class _RecordingLib:

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        proto = _lib.PROTOTYPES[name]

        def fn(*args):
            assert len(args) == len(proto), (name, len(args), len(proto))
            for a, ty in zip(args, proto):
                ty.from_param(a)  # raises on a type ctypes could not marshal
            self.calls.append(name)
            return 0

        return fn


@pytest.fixture
def dry(monkeypatch):
    rec = _RecordingLib()
    monkeypatch.setattr(ops, 'lib', lambda: rec)
    monkeypatch.setattr(ops, 'require_cuda', lambda: None)
    monkeypatch.setattr(ops, 'compute_device', lambda *t: torch.device('cpu'))
    monkeypatch.setattr(ops, 'stream_ptr', lambda: 0)
    yield rec


@pytest.fixture
def hpc_shim(monkeypatch):
    """install_hpc_rll() with ding.enable_hpc_rl set and the wrapper's cache empty; every hpc_rll module and the cache are
    put back as they were on exit"""
    from oracle import ref_loader
    ref_loader.load()
    import ding
    import ding.hpc_rl.wrapper as hw
    saved = {k: v for k, v in sys.modules.items() if k == 'hpc_rll' or k.startswith('hpc_rll.')}
    saved_fns = dict(hw.hpc_fns)
    for k in saved:
        del sys.modules[k]
    monkeypatch.setattr(ding, 'enable_hpc_rl', True)
    hw.hpc_fns.clear()
    try:
        b2.install_hpc_rll()
        yield hw
    finally:
        for k in [k for k in sys.modules if k == 'hpc_rll' or k.startswith('hpc_rll.')]:
            del sys.modules[k]
        sys.modules.update(saved)
        hw.hpc_fns.clear()
        hw.hpc_fns.update(saved_fns)


@need_ref
def test_reference_rnn_imports_with_the_hpc_switch_on(hpc_shim):
    with ref_scatter.network():
        rnn = importlib.import_module(ref_scatter.PACKAGE + '.rnn')
        assert rnn.HPCLSTM is sys.modules['hpc_rll.torch_utils.network.rnn'].LSTM
        with pytest.raises(NotImplementedError, match="'normal', 'pytorch' or 'gru'"):
            rnn.get_lstm('hpc', 8, 16, seq_len=4, batch_size=2)
    assert ref_scatter.PACKAGE + '.rnn' not in sys.modules and 'treetensor' not in sys.modules


@need_ref
def test_live_hpc_wrapper_dispatches_scatter_connection_into_the_shim(hpc_shim, dry):
    B, M, N, H, W = 2, 24, 32, 2, 3
    x, (loc, ) = make_inputs(_case(21, B, M, N, H, W))
    with reference_cls() as Ref:
        for scatter_type in ('add', 'cover'):
            model = Ref(scatter_type)
            name = 'ScatterConnection_%d_%d_%d_%d_%d_%s' % (B, M, N, H, W, scatter_type)
            dry.calls.clear()
            out = model(x, (H, W), loc)
            assert out.shape == (B, N, H, W) and dry.calls == ['b200rl_scatter_fwd']
            assert name in hpc_shim.hpc_fns['ScatterConnection']
            op = hpc_shim.hpc_fns['ScatterConnection'][name]
            assert type(op) is sys.modules['hpc_rll.torch_utils.network.scatter_connection'].ScatterConnection
            assert op.shape == (B, M, N, H, W, scatter_type)
            model(x=x, spatial_size=(H, W), location=loc)
            model(x, (H, W), location=loc)
            model(x, spatial_size=(H, W), location=loc)
            assert dry.calls == ['b200rl_scatter_fwd'] * 4
            assert hpc_shim.hpc_fns['ScatterConnection'][name] is op  # the cached instance is reused
        xr = x.clone().requires_grad_(True)
        model(xr, (H, W), loc).sum().backward()
        assert dry.calls[-2:] == ['b200rl_scatter_fwd', 'b200rl_scatter_bwd'] and xr.grad.shape == x.shape
    assert len(hpc_shim.hpc_fns['ScatterConnection']) == 2


@need_ref
def test_install_patches_the_reference_class_and_uninstall_restores_it(dry):
    B, M, N, H, W = 2, 6, 4, 3, 5
    x, (loc, ) = make_inputs(_case(22, B, M, N, H, W))
    with reference_cls() as Ref:
        forward, xy_forward = Ref.__dict__['forward'], Ref.__dict__['xy_forward']
        early = Ref('add')
        try:
            done = b2.install()
            assert (ref_scatter.PACKAGE + '.scatter_connection.ScatterConnection', 'forward') in done
            assert (ref_scatter.PACKAGE + '.scatter_connection.ScatterConnection', 'xy_forward') in done
            assert Ref.forward is sc.scatter_forward and Ref.xy_forward is sc.scatter_xy_forward
            assert not [d for d in b2.install() if 'ScatterConnection' in d[0]]  # a second call patches nothing
            dry.calls.clear()
            assert early(x, (H, W), loc).shape == (B, N, H, W)
            assert early.xy_forward(x, (H, W), loc[..., 0], loc[..., 1]).shape == (B, N, H, W)
            assert dry.calls == ['b200rl_scatter_fwd'] * 2
        finally:
            b2.uninstall()
        assert Ref.__dict__['forward'] is forward and Ref.__dict__['xy_forward'] is xy_forward


def test_dtypes_and_shapes_are_checked_before_any_launch(dry):
    x, (loc, ) = make_inputs(_case(23, 2, 5, 3, 4, 4))
    m = b2.ScatterConnection('add')
    with pytest.raises(TypeError):
        m(x.double(), (4, 4), loc)
    with pytest.raises(TypeError):
        m(x.bfloat16(), (4, 4), loc)
    with pytest.raises(TypeError):
        m(x, (4, 4), loc.int())
    with pytest.raises(TypeError):
        m.xy_forward(x, (4, 4), loc[..., 0].float(), loc[..., 1])
    with pytest.raises(TypeError):
        m.xy_forward(x, (4, 4), loc[..., 0], loc[..., 1].int())
    with pytest.raises(ValueError):
        m(x, (4, 4), loc[:, :4])
    with pytest.raises(AssertionError):
        b2.ScatterConnection('max')
    assert dry.calls == []


@pytest.mark.parametrize('bad', [(0, -1), (3, 4), (4, 0), (-1, 2)])
def test_out_of_range_index_raises_index_error_when_checking(dry, monkeypatch, bad):
    """(3, 4) is one past the last cell of a 4 x 4 map and (4, 0) a row below it; the (y, W) wrap of a row above the last
    is valid, (0, -1) is index -1"""
    monkeypatch.setattr(ops, 'CHECK_INDICES', True)
    x, (loc, ) = make_inputs(_case(24, 2, 5, 3, 4, 4))
    loc[1, 3] = torch.tensor(bad)
    for scatter_type in ('add', 'cover'):
        with pytest.raises(IndexError):
            b2.ScatterConnection(scatter_type)(x, (4, 4), loc)
        with pytest.raises(IndexError):
            b2.ScatterConnection(scatter_type).xy_forward(x, (4, 4), loc[..., 0], loc[..., 1])
    assert dry.calls == []
    loc[1, 3] = torch.tensor([2, 4])  # wraps to (3, 0)
    b2.ScatterConnection('add')(x, (4, 4), loc)
    assert dry.calls == ['b200rl_scatter_fwd']


def _transposed(B, N, H, W, seed=99):
    """an upstream gradient (B, N, H, W) laid out as the transpose of (B, N, W, H): what ``out.transpose(2, 3)`` sends back"""
    return torch.randn(B, N, W, H, generator=torch.Generator().manual_seed(seed)).transpose(2, 3)


@pytest.mark.parametrize('form', ['w1_transposed', 'h1_transposed', 'expanded', 'transposed'])
def test_backward_passes_the_cell_stride_of_the_merged_map(monkeypatch, form):
    """the backward launch gets g's strides as (B, N, H*W): g itself whenever H and W merge into one stride -- at W = 1 the
    cells step by stride(2), not by the size-1 dim's stride(3) -- and a dense copy only when they do not"""
    seen = []

    class Lib:

        def b200rl_scatter_bwd(self, *args):
            seen.append(args)
            return 0

    monkeypatch.setattr(ops, 'lib', lambda: Lib())
    monkeypatch.setattr(ops, 'stream_ptr', lambda: 0)
    B, N, M = 2, 3, 4
    H, W = {'w1_transposed': (5, 1), 'h1_transposed': (1, 5), 'expanded': (4, 6), 'transposed': (4, 6)}[form]
    g = torch.zeros(()).expand(B, N, H, W) if form == 'expanded' else _transposed(B, N, H, W)
    idx = torch.zeros(B, M, dtype=torch.int64)
    ops.scatter_bwd_(g, idx, idx, M, H, W)
    args = seen[0]
    want = {'w1_transposed': (N * H, H, 1), 'h1_transposed': (N * W, W, 1), 'expanded': (0, 0, 0),
            'transposed': (N * H * W, H * W, 1)}[form]
    assert tuple(args[1:4]) == want
    assert (args[0] == g.data_ptr()) == (form != 'transposed')


def test_fixtures_cover_every_golden_case():
    assert sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN_DIR, '*.npz'))) == sorted(GOLDEN_CASES)


@pytest.mark.parametrize('name', GOLDEN_CASES)
def test_fixture_inputs_are_the_seeded_ones(name):
    z = np.load(os.path.join(GOLDEN_DIR, name + '.npz'))
    c = golden_case(name)
    assert json.loads(str(z['case'])) == c
    x, index = make_inputs(c)
    assert np.array_equal(input_sums(x, index), z['in_sums'])
    assert np.array_equal(upstream(c).double().sum().numpy(), z['g_sum'])


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def _exact(want, got, what):
    assert want.shape == got.shape, (what, want.shape, got.shape)
    bad = np.argwhere(want.view(np.uint32) != got.view(np.uint32))
    assert not len(bad), '%s: %d of %d differ, first at %s: want %r got %r' % (
        what, len(bad), want.size, bad[0], want[tuple(bad[0])], got[tuple(bad[0])])


@gpu
@need_ref
@pytest.mark.parametrize('scatter_type', ['add', 'cover'])
@pytest.mark.parametrize('name', sorted(CASES))
def test_gpu_bit_identical_to_the_cpu_reference(name, scatter_type):
    c = CASES[name]
    x, index = make_inputs(c)
    g = upstream(c)
    with reference_cls() as Ref:
        want = run(Ref(scatter_type), c, x, index, g, 'cpu')
    got = run(b2.ScatterConnection(scatter_type), c, x, index, g, 'cuda')
    _exact(want[0], got[0], 'out')
    _exact(want[1], got[1], 'grad_x')


@gpu
@need_ref
@pytest.mark.parametrize('scatter_type', ['add', 'cover'])
def test_gpu_strided_views_read_in_place(scatter_type):
    """x permuted (n not contiguous) and sliced, location a permuted view; the same bits as contiguous copies"""
    B, M, N, H, W = 5, 300, 40, 9, 11
    gen = torch.Generator().manual_seed(31)
    x = torch.randn(B, 2 * N + 1, M, generator=gen)[:, 1::2, :].transpose(1, 2)  # (B, M, N), strides (., 1, 2M)
    loc = torch.stack([torch.randint(0, H, (B, M), generator=gen), torch.randint(0, W, (B, M), generator=gen)])
    loc = loc.permute(1, 2, 0)  # (B, M, 2), strides (M, 1, B*M)
    c = _case(0, B, M, N, H, W)
    g = upstream(c)
    with reference_cls() as Ref:
        want = run(Ref(scatter_type), c, x.contiguous(), (loc.contiguous(), ), g, 'cpu')
    xd, ld = x.cuda(), loc.cuda()
    assert not xd.is_contiguous() and not ld.is_contiguous()
    xd.requires_grad_(True)
    out = b2.ScatterConnection(scatter_type)(xd, (H, W), ld)
    out.backward(g.cuda().transpose(2, 3).contiguous().transpose(2, 3))  # a gradient whose cells have no single stride
    _exact(want[0], out.detach().cpu().numpy(), 'out')
    _exact(want[1], xd.grad.cpu().numpy(), 'grad_x')
    with reference_cls() as Ref:
        want = Ref(scatter_type).xy_forward(x, (H, W), loc[..., 0], loc[..., 1])
    got = b2.ScatterConnection(scatter_type).xy_forward(xd.detach(), (H, W), ld[..., 0], ld[..., 1])
    _exact(want.numpy(), got.cpu().numpy(), 'xy_forward')


@gpu
@need_ref
@pytest.mark.parametrize('scatter_type', ['add', 'cover'])
@pytest.mark.parametrize('H, W, M', [(40, 1, 10), (40, 1, 3), (1, 40, 10), (1, 40, 3)])
def test_gpu_single_row_or_column_map_with_a_transposed_gradient(H, W, M, scatter_type):
    """a (H, 1) or (1, W) map whose upstream gradient arrives transposed; M = 10 takes the backward's staged-tile form
    (M * 8 >= H * W), M = 3 its gather form"""
    B, N = 3, 6
    x, (loc, ) = make_inputs(_case(51, B, M, N, H, W))
    g = _transposed(B, N, H, W)
    with reference_cls() as Ref:
        xr = x.clone().requires_grad_(True)
        want = Ref(scatter_type)(xr, (H, W), loc)
        want.backward(g)
    xd = x.cuda().requires_grad_(True)
    out = b2.ScatterConnection(scatter_type)(xd, (H, W), loc.cuda())
    out.backward(g.cuda())
    _exact(want.detach().numpy(), out.detach().cpu().numpy(), 'out')
    _exact(xr.grad.numpy(), xd.grad.cpu().numpy(), 'grad_x')


@gpu
@need_ref
@pytest.mark.parametrize('name', ['hpc', 'football', 'many_per_cell'])
def test_gpu_against_the_cuda_reference(name):
    """the reference on the same CUDA tensors: its atomics reorder the 'add' sums and pick any entity of a 'cover' cell"""
    c = CASES[name]
    x, (loc, ) = make_inputs(c)
    x, loc, g = x.cuda(), loc.cuda(), upstream(c).cuda()
    idx = loc[..., 1] + loc[..., 0] * c['W']
    count = torch.zeros(c['B'], c['H'] * c['W'], dtype=torch.int64, device='cuda').scatter_add_(1, idx, torch.ones_like(idx))
    single = (count <= 1).view(c['B'], 1, c['H'], c['W']).expand(-1, c['N'], -1, -1)
    for scatter_type in ('add', 'cover'):
        with reference_cls() as Ref:
            want = run(Ref(scatter_type), c, x, (loc, ), g, 'cuda')
        got = run(b2.ScatterConnection(scatter_type), c, x, (loc, ), g, 'cuda')
        if scatter_type == 'add':
            np.testing.assert_allclose(got[0], want[0], rtol=1e-5, atol=1e-5 * np.abs(want[0]).max())
        else:
            m = single.cpu().numpy()
            _exact(want[0][m], got[0][m], 'cover out, single-entity cells')
        _exact(want[1], got[1], 'grad_x')


@gpu
@pytest.mark.parametrize('name', ['hpc', 'many_per_cell', 'chunks'])
def test_gpu_two_runs_are_bit_identical(name):
    c = CASES[name]
    x, index = make_inputs(c)
    g = upstream(c)
    for scatter_type in ('add', 'cover'):
        a = run(b2.ScatterConnection(scatter_type), c, x, index, g, 'cuda')
        b = run(b2.ScatterConnection(scatter_type), c, x, index, g, 'cuda')
        _exact(a[0], b[0], 'out')
        _exact(a[1], b[1], 'grad_x')


@gpu
@need_ref
@pytest.mark.parametrize('dense', [True, False])
def test_gpu_out_of_range_entities_are_dropped_without_checking(dense):
    """with checking off an entity whose flat index is outside [0, H*W) writes nothing and gets a zero gradient: the map is
    the reference's without those entities.  ``dense`` picks the backward's staged-tile form, else its gather form."""
    B, M, N, H, W = 4, (200 if dense else 12), 20, 10, 12
    x, (loc, ) = make_inputs(_case(41, B, M, N, H, W))
    gen = torch.Generator().manual_seed(42)
    bad = torch.rand(B, M, generator=gen) < 0.2
    bad[0, 0] = bad[1, -1] = True
    kinds = torch.randint(0, 4, (B, M), generator=gen)
    loc = loc.clone()
    loc[..., 0] = torch.where(bad & (kinds == 0), torch.full_like(loc[..., 0], H), loc[..., 0])  # a row below the map
    loc[..., 0] = torch.where(bad & (kinds == 1), torch.full_like(loc[..., 0], -1), loc[..., 0])  # index < 0
    loc[..., :] = torch.where((bad & (kinds == 2)).unsqueeze(-1), torch.tensor([0, -1]), loc)  # index -1
    loc[..., :] = torch.where((bad & (kinds == 3)).unsqueeze(-1), torch.tensor([H - 1, W]), loc)  # one past the last cell
    g = upstream(_case(0, B, M, N, H, W))
    xd = x.cuda().requires_grad_(True)
    for scatter_type in ('add', 'cover'):
        out = b2.ScatterConnection(scatter_type)(xd, (H, W), loc.cuda())
        out.backward(g.cuda())
        with reference_cls() as Ref:
            for b in range(B):
                keep = ~bad[b]
                xb = x[b:b + 1, keep].clone().requires_grad_(True)
                want = Ref(scatter_type)(xb, (H, W), loc[b:b + 1, keep])
                want.backward(g[b:b + 1])
                _exact(want.detach().numpy(), out[b:b + 1].detach().cpu().numpy(), 'out[%d]' % b)
                gx = xd.grad[b].cpu()
                _exact(xb.grad[0].numpy(), gx[keep].numpy(), 'grad_x[%d]' % b)
                assert not gx[bad[b]].any()
        xd.grad = None


@gpu
@pytest.mark.parametrize('name', GOLDEN_CASES)
def test_gpu_matches_the_fixtures(name):
    z = np.load(os.path.join(GOLDEN_DIR, name + '.npz'))
    c = golden_case(name)
    x, index = make_inputs(c)
    for scatter_type in ('add', 'cover'):
        got = run(b2.ScatterConnection(scatter_type), c, x, index, upstream(c), 'cuda')
        for k, v in zip(('out', 'grad_x'), got):
            s, total = sample(v)
            _exact(z['%s_%s' % (scatter_type, k)], s, '%s %s' % (scatter_type, k))
            if total is not None:
                assert total == z['%s_%s_sum' % (scatter_type, k)], k


@gpu
@pytest.mark.parametrize('backend', ['aot_eager', 'inductor'])
def test_gpu_fullgraph_compile_matches_eager(backend):
    """ScatterConnection -> conv2d -> mean, traced without a graph break; bit-identical to eager mode where the graph runs
    the same kernels (aot_eager), within 1e-6 where inductor writes its own reduction"""
    c = CASES['football']
    x, (loc, ) = make_inputs(dict(c, B=8))
    torch.manual_seed(0)
    conv = torch.nn.Conv2d(c['N'], 4, 3, padding=1).cuda()
    model = b2.ScatterConnection('add')

    def step(x, loc):
        return conv(model(x, (c['H'], c['W']), loc)).mean()

    torch._dynamo.reset()
    compiled = torch.compile(step, fullgraph=True, backend=backend)
    res = []
    for fn in (step, compiled):
        xd = x.cuda().requires_grad_(True)
        conv.zero_grad()
        loss = fn(xd, loc.cuda())
        loss.backward()
        res.append([loss.detach().cpu(), xd.grad.cpu(), conv.weight.grad.cpu()])
    for a, b in zip(*res):
        if backend == 'aot_eager':
            assert torch.equal(a, b)
        else:
            torch.testing.assert_close(b, a, rtol=1e-6, atol=1e-6 * float(a.abs().max()))


@gpu
@need_ref
def test_gpu_ported_reference_unit_tests():
    """ding/torch_utils/network/tests/test_scatter.py, on CUDA tensors (its keyword call form and xy_forward), against the
    reference on the CPU"""
    for scatter_type in ['add', 'cover']:
        torch.manual_seed(0)
        model = b2.ScatterConnection(scatter_type)
        B, M, N = 2, 24, 32
        H, W = 2, 3
        inp = torch.rand(B, M, N).requires_grad_(True)
        h = torch.randint(low=0, high=H, size=(B, M)).unsqueeze(dim=2)
        w = torch.randint(low=0, high=W, size=(B, M)).unsqueeze(dim=2)
        location = torch.cat([h, w], dim=2)
        xd = inp.detach().cuda().requires_grad_(True)
        output = model(x=xd, spatial_size=(H, W), location=location.cuda())
        output.mean().backward()
        assert isinstance(xd.grad, torch.Tensor)
        with reference_cls() as Ref:
            want = Ref(scatter_type)(x=inp, spatial_size=(H, W), location=location)
            want.mean().backward()
        _exact(want.detach().numpy(), output.detach().cpu().numpy(), 'naive out')
        _exact(inp.grad.numpy(), xd.grad.cpu().numpy(), 'naive grad')

        B, M, N = 10, 20, 3
        spatial_size = (13, 17)
        inp = torch.randn(size=(B, M, N)).requires_grad_(True)
        coord_x = torch.randint(low=0, high=13, size=(B, M))
        coord_y = torch.randint(low=0, high=17, size=(B, M))
        xd = inp.detach().cuda().requires_grad_(True)
        output = model.xy_forward(xd, spatial_size, coord_x.cuda(), coord_y.cuda())
        output.mean().backward()
        assert isinstance(xd.grad, torch.Tensor)
        assert output.shape == (B, N, *spatial_size)
        with reference_cls() as Ref:
            want = Ref(scatter_type).xy_forward(inp, spatial_size, coord_x, coord_y)
            want.mean().backward()
        _exact(want.detach().numpy(), output.detach().cpu().numpy(), 'xy out')
        _exact(inp.grad.numpy(), xd.grad.cpu().numpy(), 'xy grad')


@gpu
def test_gpu_host_tensors_come_back_on_the_host():
    c = CASES['b1']
    x, (loc, ) = make_inputs(c)
    x.requires_grad_(True)
    out = b2.ScatterConnection('add')(x, (c['H'], c['W']), loc)
    assert out.device.type == 'cpu'
    out.backward(upstream(c))
    assert x.grad.device.type == 'cpu'
    want = run(b2.ScatterConnection('add'), c, x.detach(), (loc, ), upstream(c), 'cuda')
    _exact(want[0], out.detach().numpy(), 'out')
    _exact(want[1], x.grad.numpy(), 'grad_x')
