"""The C-ABI launch sequence of the autograd wrappers whose forward launch also writes gradients, pinned on the CPU.

Those wrappers share one scheme: the forward launch writes the gradients for the upstream gradients it expects (a
device-resident record per call-site kind), and the backward launch verifies them on the device, recomputing on a
mismatch.  The first backward after such a forward hands the forward's buffers to autograd; any other backward writes
into fresh buffers and forces the recompute.

Each case below runs public ``rl_utils`` functions (``ops.PPOFunction`` / ``ops.GAEPPOFunction`` directly) against a stand-in
for the CUDA library that computes nothing and logs every call: the entry point, the name its ``_lib.check`` reports, and
every argument -- ``None`` for a null pointer, a label for any other pointer (``p0``, ``p1``, ... in the order the
addresses first appear in the case) and the exact value of every int and float.  The labels show whether a verifying
launch writes into the buffers the forward launch was given or into fresh ones, and which record (``g_hint``) each launch
reads.  Every tensor whose address is taken stays alive until its case ends, so no address is reused inside a case.

``tests/golden/launch_log.json`` holds the expected log; ``python tests/golden/make_launch_log.py`` rewrites it.
"""
import contextlib
import json
import os

import pytest
import torch

import di_engine_b200 as b2
from di_engine_b200 import _lib, ops
from tests.test_reference_suite import _RecordingLib

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'launch_log.json')
api = b2.rl_utils


class _LoggingLib:
    """_RecordingLib (every argument marshals to its ctypes prototype) that also logs each call; the ``*_supported``
    queries answer ``supported``"""

    def __init__(self, supported):
        self.rec = _RecordingLib()
        self.supported = supported
        self.log = []
        self.labels = {}

    def _arg(self, a, ty):
        if ty is not _lib.P:
            return a
        if not a:
            return None
        return self.labels.setdefault(a, 'p%d' % len(self.labels))

    def __getattr__(self, name):
        fn = getattr(self.rec, name)
        proto = _lib.PROTOTYPES[name]

        def logged(*args):
            rc = fn(*args)
            self.log.append({'fn': name, 'check': None, 'args': [self._arg(a, ty) for a, ty in zip(args, proto)]})
            return self.supported if name.endswith('_supported') else rc

        return logged


# ---------------------------------------------------------------------------------------------------------------------
# the losses: each returns its differentiable outputs in order
# ---------------------------------------------------------------------------------------------------------------------
B, N, D, NSTEP = 4, 5, 3, 3


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _rg(t):
    return t.requires_grad_(True)


def _ppo_inputs(g):
    ln = _rg(torch.randn(B, N, generator=g))
    lo = torch.randn(B, N, generator=g)
    act = torch.randint(0, N, (B, ), generator=g)
    vn = _rg(torch.randn(B, generator=g))
    vo, adv, ret = (torch.randn(B, generator=g) for _ in range(3))
    factor = torch.rand(B, 1, generator=g)
    return ln, lo, act, vn, vo, adv, ret, factor


def _ppo_error(g):
    ln, lo, act, vn, vo, adv, ret, _ = _ppo_inputs(g)
    return api.ppo_error(api.ppo_data(ln, lo, act, vn, vo, adv, ret, None, None))[0]


def _ppo_policy_error(g):
    ln, lo, act, _, _, adv, _, _ = _ppo_inputs(g)
    return api.ppo_policy_error(api.ppo_policy_data(ln, lo, act, adv, None, None))[0]


def _happo_error(g):
    ln, lo, act, vn, vo, adv, ret, factor = _ppo_inputs(g)
    return api.happo_error(api.happo_data(ln, lo, act, vn, vo, adv, ret, None, factor))[0]


def _happo_policy_error(g):
    ln, lo, act, _, _, adv, _, factor = _ppo_inputs(g)
    return api.happo_policy_error(api.happo_policy_data(ln, lo, act, adv, None, factor))[0]


def _ppo_function(g):
    ln, lo, act, vn, vo, adv, ret, _ = _ppo_inputs(g)
    return ops.PPOFunction.apply(ln, vn, lo, act, vo, adv, ret, None, None, B, 1, N, 0.2, 1, 0.0, 1, 'ppo', None)[:4]


def _gae_ppo_function(g):
    T = 2
    ln = _rg(torch.randn(T * B, N, generator=g))
    lo = torch.randn(T * B, N, generator=g)
    act = torch.randint(0, N, (T * B, ), generator=g)
    vn = _rg(torch.randn(T * B, generator=g))
    vo, ret = torch.randn(T * B, generator=g), torch.randn(T * B, generator=g)
    value, next_value, reward = (torch.randn(T, B, generator=g) for _ in range(3))
    done = torch.zeros(T, B)
    return ops.GAEPPOFunction.apply(ln, vn, value, next_value, reward, done, None, lo, act, vo, ret, None, None, T, B, N,
                                    0.99, 0.95, 0.2, 1, 0.0, 1)[1:5]


def _vtrace(g):
    T = 3
    tgt = _rg(torch.randn(T, B, N, generator=g))
    beh = torch.randn(T, B, N, generator=g)
    act = torch.randint(0, N, (T, B), generator=g)
    value = _rg(torch.randn(T + 1, B, generator=g))
    reward = torch.randn(T, B, generator=g)
    return api.vtrace_error_discrete_action(api.vtrace_data(tgt, beh, act, value, reward, None))


def _a2c(g):
    logit = _rg(torch.randn(B, N, generator=g))
    act = torch.randint(0, N, (B, ), generator=g)
    value = _rg(torch.randn(B, generator=g))
    adv, ret = torch.randn(B, generator=g), torch.randn(B, generator=g)
    return api.a2c_error(api.a2c_data(logit, act, value, adv, ret, None))


def _gauss(g, grad):
    mu, sigma = torch.randn(B, D, generator=g), torch.rand(B, D, generator=g) + 0.5
    return {'mu': _rg(mu), 'sigma': _rg(sigma)} if grad else {'mu': mu, 'sigma': sigma}


def _cont_inputs(g):
    new, old = _gauss(g, True), _gauss(g, False)
    act = torch.randn(B, D, generator=g)
    vn = _rg(torch.randn(B, generator=g))
    vo, adv, ret = (torch.randn(B, generator=g) for _ in range(3))
    factor = torch.rand(B, 1, generator=g)
    return new, old, act, vn, vo, adv, ret, factor


def _a2c_continuous(g):
    new, _, act, vn, _, adv, ret, _ = _cont_inputs(g)
    return api.a2c_error_continuous(api.a2c_data(new, act, vn, adv, ret, None))


def _ppo_error_continuous(g):
    new, old, act, vn, vo, adv, ret, _ = _cont_inputs(g)
    return api.ppo_error_continuous(api.ppo_data(new, old, act, vn, vo, adv, ret, None, None))[0]


def _ppo_policy_error_continuous(g):
    new, old, act, _, _, adv, _, _ = _cont_inputs(g)
    return api.ppo_policy_error_continuous(api.ppo_policy_data_continuous(new, old, act, adv, None, None))[0][:2]


def _happo_error_continuous(g):
    new, old, act, vn, vo, adv, ret, factor = _cont_inputs(g)
    return api.happo_error_continuous(api.happo_data(new, old, act, vn, vo, adv, ret, None, factor))[0]


def _happo_policy_error_continuous(g):
    new, old, act, _, _, adv, _, _ = _cont_inputs(g)
    return api.happo_policy_error_continuous((new, old, act, adv, None))[0]


def _q_inputs(g, shape, rows=(B, )):
    q = _rg(torch.randn(*shape, generator=g))
    nq = torch.randn(*shape, generator=g)
    act = torch.randint(0, N, rows, generator=g)
    nact = torch.randint(0, N, rows, generator=g)
    reward = torch.randn(NSTEP, B, generator=g)
    done = (torch.rand(B, generator=g) < 0.3).float()
    return q, nq, act, nact, reward, done


def _q_nstep(g):
    return api.q_nstep_td_error(api.q_nstep_td_data(*_q_inputs(g, (B, N)), None), 0.95, nstep=NSTEP)


def _bdq_nstep(g):
    return api.bdq_nstep_td_error(api.q_nstep_td_data(*_q_inputs(g, (B, D, N), (B, D)), None), 0.95, nstep=NSTEP)


def _dqfd(g):
    q, nq, act, nact, reward, done = _q_inputs(g, (B, N))
    nq1, nact1 = torch.randn(B, N, generator=g), torch.randint(0, N, (B, ), generator=g)
    expert = (torch.rand(B, generator=g) < 0.5).float()
    data = api.dqfd_nstep_td_data(q, nq, act, nact, reward, done, done, None, nq1, nact1, expert)
    loss, per, stats = api.dqfd_nstep_td_error(data, 0.95, 1.0, 1.0, 0.8, nstep=NSTEP)
    return (loss, per) + tuple(stats)


def _m_q(g):
    q, nq, act, _, reward, done = _q_inputs(g, (B, N))
    tq = torch.randn(B, N, generator=g)
    return api.m_q_1step_td_error(api.m_q_1step_td_data(q, tq, nq, act, reward[0], done, None), 0.99, 0.03, 0.9)[:2]


def _sql(g):
    return api.q_nstep_sql_td_error(api.q_nstep_td_data(*_q_inputs(g, (B, N)), None), 0.99, 0.1, nstep=NSTEP)[:2]


def _q_v(g):
    q, _, act, _, reward, done = _q_inputs(g, (B, N))
    v = torch.randn(B, generator=g)
    return api.q_v_1step_td_error(api.q_v_1step_td_data(q, v, act, reward[0], done, None), 0.99)


def _qrdqn(g):
    q, nq, act, nact, reward, done = _q_inputs(g, (B, N, 3))
    return api.qrdqn_nstep_td_error(api.qrdqn_nstep_td_data(q, nq, act, nact, reward, done, 3, None), 0.95, nstep=NSTEP)


def _iqn(g):
    q, nq, act, nact, reward, done = _q_inputs(g, (3, B, N))
    tau = torch.rand(3, B, 1, generator=g)
    return api.iqn_nstep_td_error(api.iqn_nstep_td_data(q, nq, act, nact, reward, done, tau, None), 0.95, nstep=NSTEP)


def _fqf(g):
    q, nq, act, nact, reward, done = _q_inputs(g, (B, 3, N))
    tau = torch.rand(B, 3, generator=g)
    return api.fqf_nstep_td_error(api.fqf_nstep_td_data(q, nq, act, nact, reward, done, tau, None), 0.95, nstep=NSTEP)


def _c51(g):
    dist = _rg(torch.rand(B, N, 11, generator=g) + 0.1)
    ndist = torch.rand(B, N, 11, generator=g) + 0.1
    _, _, act, nact, reward, done = _q_inputs(g, (B, N))
    data = api.dist_nstep_td_data(dist, ndist, act, nact, reward, done, None)
    return api.dist_nstep_td_error(data, 0.95, -10.0, 10.0, 11, NSTEP)


def _upgo(g):
    T = 3
    logit = _rg(torch.randn(T, B, N, generator=g))
    act = torch.randint(0, N, (T, B), generator=g)
    rhos, rewards = torch.randn(T, B, generator=g), torch.randn(T, B, generator=g)
    return (api.upgo_loss(logit, rhos, act, rewards, torch.randn(T + 1, B, generator=g)), )


# name -> (loss, default upstream weights, a different mix); the policy-gradient defaults are the learners' loss weights
# (policy 1, value 0.5, entropy -0.01, no KL term); a TD loss is back-propagated alone
PG = {
    'ppo_error': (_ppo_error, [1.0, 0.5, -0.01], [0.7, 2.0, 0.05, -1.5]),
    'ppo_policy_error': (_ppo_policy_error, [1.0, -0.01], [0.7, 0.05, -1.5]),
    'happo_error': (_happo_error, [1.0, 0.5, -0.01], [0.7, 2.0, 0.05]),
    'happo_policy_error': (_happo_policy_error, [1.0, -0.01], [0.7, 0.05]),
    'ppo_function': (_ppo_function, [1.0, 0.5, -0.01], [0.7, 2.0, 0.05, -1.5]),
    'gae_ppo_function': (_gae_ppo_function, [1.0, 0.5, -0.01], [0.7, 2.0, 0.05, -1.5]),
    'vtrace': (_vtrace, [1.0, 0.5, -0.01], [0.7, 2.0, 0.05]),
    'a2c': (_a2c, [1.0, 0.5, -0.01], [0.7, 2.0, 0.05]),
    'a2c_continuous': (_a2c_continuous, [1.0, 0.5, -0.01], [0.7, 2.0, 0.05]),
    'ppo_error_continuous': (_ppo_error_continuous, [1.0, 0.5, -0.01], [0.7, 2.0, 0.05, -1.5]),
    'ppo_policy_error_continuous': (_ppo_policy_error_continuous, [1.0, -0.01], [0.7, 0.05]),
    'happo_error_continuous': (_happo_error_continuous, [1.0, 0.5, -0.01], [0.7, 2.0, 0.05]),
    'happo_policy_error_continuous': (_happo_policy_error_continuous, [1.0, -0.01], [0.7, 0.05]),
    'upgo': (_upgo, [1.0], [0.5]),
}
TD = {
    'q_nstep': _q_nstep, 'bdq_nstep': _bdq_nstep, 'dqfd': _dqfd, 'm_q': _m_q, 'sql': _sql, 'q_v': _q_v, 'qrdqn': _qrdqn,
    'iqn': _iqn, 'fqf': _fqf, 'c51': _c51,
}
FUSED_QUERY = ('ppo_error', 'ppo_policy_error', 'happo_error', 'happo_policy_error', 'ppo_function', 'vtrace')


def _backward(outs, weights, twice=False):
    total = sum(w * o for w, o in zip(weights, outs))
    total.backward(retain_graph=twice)
    if twice:
        total.backward()


def _schedule(loss, weights, mix, sched):
    if sched == 'no_grad':
        with torch.no_grad():
            loss(_g(1))
    else:
        _backward(loss(_g(1)), mix if sched == 'mix' else weights, sched == 'twice')


def _per_sample(loss):
    outs = loss(_g(1))
    total = outs[0] + sum((o * torch.linspace(0.5, 1.5, o.numel()).reshape(o.shape)).sum() for o in outs[1:])
    total.backward()


def _unfused(loss, weights):
    flag = 'VTRACE_FUSED' if loss is _vtrace else 'PPO_FUSED_BACKWARD'
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(ops, flag, False)
        _backward(loss(_g(1)), weights)
        _backward(loss(_g(2)), weights, twice=True)


def _alternate(*losses):
    for i, (loss, weights) in enumerate(losses):
        _backward(loss(_g(i)), weights)


def _cases():
    cases = {}
    for name, (loss, weights, mix) in PG.items():
        for sched in ('no_grad', 'default', 'mix', 'twice'):
            cases['%s-%s' % (name, sched)] = (1, lambda l=loss, w=weights, m=mix, s=sched: _schedule(l, w, m, s))
        if name in FUSED_QUERY:
            cases[name + '-unsupported'] = (0, lambda l=loss, w=weights: _backward(l(_g(1)), w))
            cases[name + '-unfused'] = (1, lambda l=loss, w=weights: _unfused(l, w))
    for name, loss in TD.items():
        for sched in ('no_grad', 'default', 'mix', 'twice'):
            cases['%s-%s' % (name, sched)] = (1, lambda l=loss, s=sched: _schedule(l, [1.0], [0.5], s))
        cases[name + '-per_sample'] = (1, lambda l=loss: _per_sample(l))
    ppoc, ppoc_policy, happoc_policy = (PG[k][:2] for k in ('ppo_error_continuous', 'ppo_policy_error_continuous',
                                                            'happo_policy_error_continuous'))
    cases['ppoc_alternating_with_its_policy_half'] = (1, lambda: _alternate(ppoc_policy, ppoc, ppoc_policy, ppoc))
    cases['ppoc_alternating_with_happo_policy_half'] = (1, lambda: _alternate(happoc_policy, ppoc, happoc_policy))
    return cases


CASES = _cases()


def record(name):
    """the launch log of case ``name``"""
    supported, body = CASES[name]
    lib = _LoggingLib(supported)
    keep = []
    data_ptr = torch.Tensor.data_ptr

    def keep_alive(t):
        keep.append(t)
        return data_ptr(t)

    def check(rc, what):
        assert rc == 0 and lib.log[-1]['check'] is None, (rc, what)
        lib.log[-1]['check'] = what

    ws = torch.zeros(1 << 18)
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(ops, 'lib', lambda: lib)
        mp.setattr(ops, 'require_cuda', lambda: None)
        mp.setattr(ops, 'compute_device', lambda *t: torch.device('cpu'))
        mp.setattr(ops, 'stream_ptr', lambda: 0)
        mp.setattr(ops, 'workspace', lambda dev: ws)
        mp.setattr(torch.cuda, 'device', lambda d: contextlib.nullcontext())
        mp.setattr(b2.rl_utils.td, 'CHECK_DIST_POSITIVE', False)
        mp.setattr(b2.rl_utils.ppo, 'LAZY_INFO', False)
        mp.setattr(_lib, 'check', check)
        mp.setattr(torch.Tensor, 'data_ptr', keep_alive)
        body()
    del keep
    return lib.log


_golden = None


def _load():
    global _golden
    if _golden is None:
        with open(GOLDEN) as f:
            _golden = json.load(f)
    return _golden


def test_every_case_has_a_recorded_log():
    assert sorted(_load()) == sorted(CASES)


@pytest.mark.filterwarnings('ignore:invalid value encountered in cast')  # the stand-in leaves outputs uninitialised
@pytest.mark.parametrize('name', sorted(CASES))
def test_launch_log(name):
    want = _load().get(name)
    assert want is not None, 'no recorded log for %s (python tests/golden/make_launch_log.py)' % name
    got = record(name)
    assert len(got) == len(want), ([e['fn'] for e in got], [e['fn'] for e in want])
    for i, (a, b) in enumerate(zip(got, want)):
        assert a == b, (i, a, b)
