"""Installing the CUDA operators into a running DI-engine.

Two routes, matching the two ways the reference reaches its operators (SURVEY.md section 8b):

* ``install()``: policies bind the operators at import time (``from ding.rl_utils import gae`` -- policy/ppo.py:8-10,
  policy/dqn.py:7, policy/c51.py:6, policy/impala.py:8 ...), so the names are rebound in ``ding.rl_utils``, its
  submodules and every already-imported ``ding.*`` / ``dizoo.*`` module that holds a reference to the original.
* ``install_hpc_rll()``: registers an ``hpc_rll`` module tree so that the reference's own plugin switch
  (``ENABLE_DI_HPC=true`` -> ding/hpc_rl/wrapper.py:61-83) constructs these operators as ``Class(*shape).cuda()``.
"""
import sys
import types

from . import rl_utils as _ours

_installed = []  # (module, name, original)


def _originals():
    """name -> set of objects that count as 'the reference implementation' of that name."""
    found = {}
    base = sys.modules.get('ding.rl_utils')
    for name in _ours.HOT_PATH_FUNCTIONS + _ours.LM_HOT_PATH_FUNCTIONS:
        objs = set()
        cands = [base] + [sys.modules.get('ding.rl_utils.' + m) for m in ('gae', 'ppo', 'td', 'vtrace', 'upgo', 'a2c', 'retrace', 'happo', 'acer', 'ppg',
                                                                          'grpo', 'rloo', 'log_prob_utils')]
        for mod in cands:
            fn = getattr(mod, name, None) if mod is not None else None
            if fn is not None and fn is not getattr(_ours, name):
                objs.add(fn)
        found[name] = objs
    return found


def install(prefixes=('ding', 'dizoo'), skip_modules=(), verbose=False):
    """Rebind the hot-path functions to the CUDA implementations. Returns the list of (module, name) rebound.

    Call it after the policy modules you use are imported (or import ``ding.policy`` first); calling it again
    picks up modules imported since.  ``skip_modules`` (exact names) are left alone -- e.g. ``'ding.rl_utils.adder'``
    to keep the collector-side CPU GAE of policy/ppo.py:541 on the reference path.
    """
    from . import ops
    ops.require_cuda()
    originals = _originals()
    done = []
    for mod_name, mod in list(sys.modules.items()):
        if mod is None or mod_name in skip_modules:
            continue
        if not any(mod_name == p or mod_name.startswith(p + '.') for p in prefixes):
            continue
        for name, objs in originals.items():
            cur = mod.__dict__.get(name)
            if cur is not None and cur in objs:
                _installed.append((mod, name, cur))
                setattr(mod, name, getattr(_ours, name))
                done.append((mod_name, name))
                if verbose:
                    print('di_engine_b200: %s.%s -> CUDA kernel' % (mod_name, name))
    return done


def uninstall():
    """Undo every rebinding made by ``install``."""
    while _installed:
        mod, name, orig = _installed.pop()
        setattr(mod, name, orig)


# ---------------------------------------------------------------------------------------------------------------
# hpc_rll-shaped shim for the reference's ENABLE_DI_HPC switch
# ---------------------------------------------------------------------------------------------------------------
class _HpcOp:
    """Callable constructed as ``Class(*shape)`` and moved with ``.cuda()`` by ding/hpc_rl/wrapper.py:75-76.
    The wrapper calls ``op(*namedtuple_fields, *scalars, **kwargs)`` (:123-125) and drops every argument that is not
    whitelisted, so sizes such as nstep / n_atom are re-derived from the tensors."""

    def __init__(self, *shape):
        self.shape = tuple(shape)

    def cuda(self, device=None):
        return self

    def to(self, *a, **k):
        return self


class GAE(_HpcOp):

    def __call__(self, value, next_value, reward, done, traj_flag, gamma=0.99, lambda_=0.97, **kw):
        lambda_ = kw.pop('lambda', lambda_)
        return _ours.gae(_ours.gae_data(value, next_value, reward, done, traj_flag), gamma, lambda_)


class PPO(_HpcOp):

    def __call__(self, logit_new, logit_old, action, value_new, value_old, adv, return_, weight,
                 logit_pretrained=None, clip_ratio=0.2, use_value_clip=True, dual_clip=None, **kw):
        data = _ours.ppo_data(logit_new, logit_old, action, value_new, value_old, adv, return_, weight,
                              logit_pretrained)
        return _ours.ppo_error(data, clip_ratio, use_value_clip, dual_clip)


class QNStepTD(_HpcOp):

    def __call__(self, q, next_n_q, action, next_n_action, reward, done, weight, gamma=0.99, **kw):
        data = _ours.q_nstep_td_data(q, next_n_q, action, next_n_action, reward, done, weight)
        return _ours.q_nstep_td_error(data, gamma, nstep=reward.shape[0])


class QNStepTDRescale(_HpcOp):

    def __call__(self, q, next_n_q, action, next_n_action, reward, done, weight, gamma=0.99, **kw):
        data = _ours.q_nstep_td_data(q, next_n_q, action, next_n_action, reward, done, weight)
        return _ours.q_nstep_td_error_with_rescale(data, gamma, nstep=reward.shape[0])


class DistNStepTD(_HpcOp):

    def __call__(self, dist, next_n_dist, act, next_n_act, reward, done, weight, gamma=0.99, v_min=-10., v_max=10.,
                 **kw):
        data = _ours.dist_nstep_td_data(dist, next_n_dist, act, next_n_act, reward, done, weight)
        return _ours.dist_nstep_td_error(data, gamma, v_min, v_max, dist.shape[-1], nstep=reward.shape[0])


class TDLambda(_HpcOp):

    def __call__(self, value, reward, weight, gamma=0.9, lambda_=0.8, **kw):
        lambda_ = kw.pop('lambda', lambda_)
        return _ours.td_lambda_error(_ours.td_lambda_data(value, reward, weight), gamma, lambda_)


class UPGO(_HpcOp):

    def __call__(self, target_output, rhos, action, rewards, bootstrap_values, mask=None, **kw):
        return _ours.upgo_loss(target_output, rhos, action, rewards, bootstrap_values, mask)


class VTrace(_HpcOp):

    def __call__(self, target_output, behaviour_output, action, value, reward, weight, gamma=0.99, lambda_=0.95,
                 rho_clip_ratio=1.0, c_clip_ratio=1.0, rho_pg_clip_ratio=1.0, **kw):
        lambda_ = kw.pop('lambda', lambda_)
        data = _ours.vtrace_data(target_output, behaviour_output, action, value, reward, weight)
        return _ours.vtrace_error_discrete_action(data, gamma, lambda_, rho_clip_ratio, c_clip_ratio,
                                                  rho_pg_clip_ratio)


_HPC_LAYOUT = {
    'hpc_rll.rl_utils.gae': {'GAE': GAE},
    'hpc_rll.rl_utils.td': {'DistNStepTD': DistNStepTD, 'QNStepTD': QNStepTD, 'QNStepTDRescale': QNStepTDRescale,
                            'TDLambda': TDLambda},
    'hpc_rll.rl_utils.ppo': {'PPO': PPO},
    'hpc_rll.rl_utils.upgo': {'UPGO': UPGO},
    'hpc_rll.rl_utils.vtrace': {'VTrace': VTrace},
}


def install_hpc_rll(force=False):
    """Register an ``hpc_rll`` package exposing the classes named in ding/hpc_rl/wrapper.py:62-73."""
    if 'hpc_rll' in sys.modules and not force and not getattr(sys.modules['hpc_rll'], '__b200_shim__', False):
        raise RuntimeError("a real hpc_rll package is already imported; pass force=True to shadow it")
    root = types.ModuleType('hpc_rll')
    root.__b200_shim__ = True
    root.__path__ = []
    sys.modules['hpc_rll'] = root
    sub = types.ModuleType('hpc_rll.rl_utils')
    sub.__path__ = []
    sys.modules['hpc_rll.rl_utils'] = sub
    root.rl_utils = sub
    for mod_name, classes in _HPC_LAYOUT.items():
        m = types.ModuleType(mod_name)
        for k, v in classes.items():
            setattr(m, k, v)
        sys.modules[mod_name] = m
        setattr(sub, mod_name.rsplit('.', 1)[1], m)
    return root
