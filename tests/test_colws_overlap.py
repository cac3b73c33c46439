"""Captured learner steps of the one-launch GAE + ppo_error column kernel (csrc/colws.cu) against the same steps run eagerly.

Inside a CUDA graph, a step's column kernel may start streaming its inputs before the previous step's finalize and check
launches have completed, where nothing it reads early is written by them (common.cuh).  Every case here runs K >= 8 steps
eagerly and then as one captured graph, and requires bit-identical results: rotated buffer sets (the overlap engages),
the same set twice in a row (in-place next_value), a step reading the previous step's outputs, a torch op between two
steps that rewrites the next step's inputs, and the autograd wrapper with a loss weight that changes on one step.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

T, B, N = 32, 4096, 6  # 4096 columns: the 32-column tiles, one per SM, as at config D
GAMMA, LAMBDA, CLIP = 0.99, 0.95, 0.2
MIX = (1.0, 0.5, -0.01)
K = 8


def _ops():
    from di_engine_b200 import ops
    return ops


def _inputs(seed, dev):
    g = torch.Generator().manual_seed(seed)
    value = torch.randn(T, B, generator=g)
    done = (torch.rand(T, B, generator=g) < 0.05).float()
    next_value = torch.where(done.bool(), torch.randn(T, B, generator=g), torch.randn(T, B, generator=g))
    traj = done.clone()
    traj[-1] = 1.0
    logit_new = torch.randn(T * B, N, generator=g)
    d = dict(value=value, next_value=next_value, reward=torch.randn(T, B, generator=g), done=done, traj_flag=traj,
             logit_new=logit_new, logit_old=logit_new + 0.1 * torch.rand(T * B, N, generator=g),
             action=torch.randint(0, N, (T * B, ), generator=g), value_new=torch.randn(T * B, generator=g),
             value_old=torch.randn(T * B, generator=g), return_=torch.randn(T * B, generator=g))
    return {k: v.to(dev) for k, v in d.items()}


class Step:
    """One learner step through the C ABI on its own buffers: the one-launch forward with gradients (+ finalize) and the
    device-verified backward check.  `alias` replaces inputs by other tensors (another step's outputs)."""

    def __init__(self, seed, dev='cuda', alias=None):
        ops = _ops()
        self.ops = ops
        self.b = _inputs(seed, dev)
        self.b.update(alias or {})
        self.init = {k: v.clone() for k, v in self.b.items()}
        self.hint = torch.tensor([MIX[0], MIX[1], MIX[2], 0.0], device=dev)
        self.g = [torch.tensor(x, device=dev) for x in MIX]
        self.g_used = torch.zeros(4, device=dev)
        self.adv = torch.zeros(T, B, device=dev)
        self.out = torch.zeros(8, device=dev)
        self.grad_logit = torch.zeros(T * B, N, device=dev)
        self.grad_value = torch.zeros(T * B, device=dev)
        self.ws = ops.workspace(torch.device(dev))

    def outputs(self):
        return dict(adv=self.adv, out=self.out, grad_logit=self.grad_logit, grad_value=self.grad_value,
                    g_used=self.g_used, hint=self.hint)

    def reset(self):
        for k, v in self.b.items():
            v.copy_(self.init[k])
        for v in self.outputs().values():
            v.zero_()
        self.hint.copy_(torch.tensor([MIX[0], MIX[1], MIX[2], 0.0]))

    def __call__(self):
        o, b, p = self.ops, self.b, self.ops.ptr
        lib = o.lib()
        rc = lib.b200rl_gae_ppo_fwd_grad(
            p(b['value']), p(b['next_value']), p(b['reward']), p(b['done']), p(b['traj_flag']), T, B, GAMMA, LAMBDA, 1,
            p(b['logit_new']), p(b['logit_old']), None, p(b['action']), p(b['value_new']), p(b['value_old']),
            p(b['return_']), None, N, CLIP, 1, 0.0, 1, p(self.hint), p(self.g_used), p(self.adv), p(self.out),
            p(self.grad_logit), p(self.grad_value), p(self.ws), self.ws.numel() * 4, o.stream_ptr())
        assert rc == 0, rc
        rc = lib.b200rl_ppo_bwd(
            p(b['logit_new']), p(b['logit_old']), None, p(b['action']), p(b['value_new']), p(b['value_old']), p(self.adv),
            p(b['return_']), None, T * B, 1, N, CLIP, 1, 0.0, 1, None, None, p(self.g[0]), p(self.g[1]), p(self.g[2]),
            None, p(self.g_used), p(self.hint), p(self.grad_logit), p(self.grad_value), o.stream_ptr())
        assert rc == 0, rc


def _snapshot(steps):
    seen, snap = set(), []
    for s in steps:
        if id(s) in seen:
            continue
        seen.add(id(s))
        snap.append({k: v.clone() for k, v in dict(s.b, **s.outputs()).items()})
    return snap


def _run(seq, between=None):
    """the K steps of `seq` eagerly, then captured as one graph and replayed on the same reset buffers: both snapshots"""
    steps = list(dict.fromkeys(seq))
    res = []
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        for graph in (False, True):
            for s in steps:
                s.reset()
            if graph:
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g, stream=stream):
                    for i, s in enumerate(seq):
                        s()
                        if between:
                            between(i)
                for s in steps:
                    s.reset()
                g.replay()
            else:
                for i, s in enumerate(seq):
                    s()
                    if between:
                        between(i)
            stream.synchronize()
            res.append(_snapshot(seq))
    return res


def _assert_same(eager, graph):
    assert len(eager) == len(graph)
    for e, g in zip(eager, graph):
        for k in e:
            assert torch.equal(e[k], g[k]), k


@pytest.mark.parametrize('nsets', [2, 4])
def test_rotated_sets(nsets):
    sets = [Step(100 + i) for i in range(nsets)]
    _assert_same(*_run([sets[i % nsets] for i in range(K)]))


def test_same_set_twice():
    s = Step(7)
    a, b = Step(8), Step(9)
    _assert_same(*_run([a, s, s, b, s, s, a, s]))


def test_next_step_reads_previous_outputs():
    a = Step(11)
    b = Step(12, alias={'value': a.adv, 'logit_old': a.grad_logit})  # b reads a's advantages and gradients
    c = Step(13, alias={'value_new': b.grad_value, 'reward': b.adv})  # c reads b's
    _assert_same(*_run([a, b, c, a, b, c, a, b, c]))


def test_torch_op_between_steps_rewrites_next_inputs():
    sets = [Step(20 + i) for i in range(2)]
    seq = [sets[i % 2] for i in range(K)]

    def between(i):
        nxt = seq[(i + 1) % K].b
        nxt['reward'].mul_(0.5).add_(0.25)
        nxt['logit_old'].add_(0.01)

    _assert_same(*_run(seq, between))


def test_autograd_step_in_graph(monkeypatch):
    import di_engine_b200 as b2
    monkeypatch.setattr(b2.rl_utils.ppo, 'LAZY_INFO', True)  # no host read of the info scalars inside the capture
    dev = 'cuda'
    batches = [_inputs(30 + i, dev) for i in range(2)]
    leaves = [(b['logit_new'].clone().requires_grad_(True), b['value_new'].clone().requires_grad_(True)) for b in batches]
    weights = [MIX] * K
    weights[3] = (1.0, 0.25, -0.01)  # the backward check recomputes on this step
    init = [{k: v.clone() for k, v in b.items()} for b in batches]

    def steps():
        res = []
        for i in range(K):
            b, (ln, vn) = batches[i % 2], leaves[i % 2]
            adv, loss, _ = b2.gae_ppo_error(
                b2.gae_data(b['value'], b['next_value'], b['reward'], b['done'], b['traj_flag']),
                b2.ppo_data(ln, b['logit_old'], b['action'], vn, b['value_old'], None, b['return_'], None, None), GAMMA,
                LAMBDA, CLIP, True, None)
            w = weights[i]
            total = w[0] * loss.policy_loss + w[1] * loss.value_loss + w[2] * loss.entropy_loss
            gl, gv = torch.autograd.grad(total, [ln, vn])
            res.append((adv, total, gl, gv))
        return res

    def reset():
        for b, i in zip(batches, init):
            for k, v in b.items():
                v.copy_(i[k])

    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        eager = [tuple(t.clone() for t in r) for r in steps()]
        stream.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=stream):
            out = steps()
        reset()
        g.replay()
        stream.synchronize()
    for e, r in zip(eager, out):
        for x, y in zip(e, r):
            assert torch.equal(x, y)
