"""di_engine_b200 -- H100 (sm_90a) learner hot path for DI-engine.

The trajectory return/advantage and policy-loss operators of ``ding.rl_utils`` (gae, td_lambda_error,
vtrace_error_discrete_action, upgo_loss, ppo_error, q_nstep_td_error, q_nstep_td_error_with_rescale,
dist_nstep_td_error, generalized_lambda_returns) as hand-written CUDA kernels behind a C ABI
(``include/b200rl.h`` -> ``lib/libb200rl.so``) with the reference's Python signatures on top (``rl_utils``).

    import di_engine_b200 as b2
    adv = b2.rl_utils.gae(b2.rl_utils.gae_data(value, next_value, reward, done, traj_flag), 0.99, 0.95)
    b2.install()            # rebinds the same names inside an imported ``ding`` (drop-in for Policy._forward_learn)

The on-disk directory is ``di-engine_b200`` (not an importable identifier); ``di_engine_b200.py`` at the repository
root loads it under the importable name.
"""
from . import _lib, collate, data, ops, parallel, rl_utils, torch_ops, torch_utils
from .collate import preprocess_learn
from .data import PackedBatch
from .installer import install, install_hpc_rll, uninstall
from .rl_utils import *  # noqa: F401,F403
from .torch_utils import ScatterConnection

__version__ = '0.1.0'


def library_path():
    return _lib.LIB_PATH


def is_built():
    import os
    return os.path.isfile(_lib.LIB_PATH)
