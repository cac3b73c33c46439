"""ctypes binding of ``lib/libb200rl.so`` -- the C ABI declared in ``include/b200rl.h``.

There is no fallback: if the shared library is missing (not built) importing the operators raises, and every
operator raises when no CUDA device is present.  Build with ``python __graft_entry__.py`` / ``make -C csrc``.
"""
import ctypes
import os
from ctypes import c_double, c_int, c_longlong, c_size_t, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
# B200RL_LIB: load another build of the same ABI (tuning experiments build variants next to the default library)
LIB_PATH = os.environ.get("B200RL_LIB") or os.path.join(_HERE, "lib", "libb200rl.so")

P = c_void_p  # device pointer
LL = c_longlong
D = c_double
I = c_int

# name -> argtypes (restype is int unless listed in _RESTYPE); mirrors include/b200rl.h one to one
PROTOTYPES = {
    "b200rl_version": [],
    "b200rl_built_for_sm": [],
    "b200rl_workspace_bytes": [],
    "b200rl_gae": [P, P, P, P, P, P, LL, LL, LL, D, D, I, P],
    "b200rl_gae_returns": [P, P, P, P, P, LL, LL, LL, D, D, I, D, P, P, P, P, P, P, P, c_size_t, P],
    "b200rl_adv_stats": [P, LL, P, P, c_size_t, P],
    "b200rl_normalize": [P, P, LL, P, P],
    "b200rl_gae_returns_norm": [P, P, P, P, P, LL, LL, D, D, I, D, P, P, P, P, P, P, P, P, P, c_size_t, P],
    "b200rl_value_map_fwd": [I, P, LL, P, P],
    "b200rl_value_map_bwd": [I, P, P, LL, P, P],
    "b200rl_impala_mask": [P, P, P, LL, LL, P, P, P, P],
    "b200rl_ppo_fwd": [P, P, P, P, P, P, P, P, P, LL, LL, LL, D, I, D, I, P, P, P, P, c_size_t, P],
    "b200rl_ppo_bwd": [P, P, P, P, P, P, P, P, P, LL, LL, LL, D, I, D, I, P, P, P, P, P, P, P, P, P, P, P],
    "b200rl_ppo_fwd_grad": [P, P, P, P, P, P, P, P, P, LL, LL, LL, D, I, D, I, P, P, P, P, P, P, P, P, c_size_t, P],
    "b200rl_ppo_value_fwd": [P, P, P, P, LL, D, I, P, P, P, c_size_t, P],
    "b200rl_ppo_fused_supported": [P, P, P, P, P, P, P, P, P, P, LL, LL],
    "b200rl_ppo_tile_geometry": [LL, LL, I, I, I, I, P],
    "b200rl_qntd_fwd": [P, P, P, P, P, P, P, P, LL, P, LL, LL, LL, I, D, I, I, D, I, D, I, LL, D, P, P, P, P, P, P, P,
                        c_size_t, P],
    "b200rl_qntd_bwd": [P, P, P, P, P, LL, LL, LL, I, LL, I, P, P],
    "b200rl_dqfd_fwd": [P, P, P, P, P, P, P, P, P, P, P, LL, P, LL, LL, I, D, I, I, D, I, D, D, D, D, D, LL, D, P, P, P,
                        P, P, P, P, P, P, c_size_t, P],
    "b200rl_dqfd_bwd": [P, P, P, P, P, P, P, P, LL, LL, D, D, D, LL, I, P, P],
    "b200rl_soft_td_fwd": [I, P, P, P, P, P, P, P, P, LL, LL, LL, LL, I, D, D, D, I, I, D, P, P, P, P, P, P, P, P, P,
                           c_size_t, P],
    "b200rl_dntd_fwd":[P, P, P, P, P, P, P, LL, P, LL, P, LL, LL, LL, I, I, D, D, D, P, P, P, P, P, P, c_size_t, P],
    "b200rl_dntd_bwd": [P, P, P, P, LL, P, P, LL, LL, I, I, P, P],
    "b200rl_lambda_returns": [P, P, P, D, P, D, P, I, LL, LL, P, P],
    "b200rl_lambda_returns_bwd": [P, P, P, P, P, D, P, D, P, I, LL, LL, P, P, P, P, P],
    "b200rl_tb_cross_entropy_fwd": [P, P, P, LL, LL, LL, P, P],
    "b200rl_tb_cross_entropy_bwd": [P, P, P, P, LL, LL, LL, P, P],
    "b200rl_td_lambda_fwd": [P, P, P, D, D, LL, LL, P, P, P, c_size_t, P],
    "b200rl_scale": [P, P, P, LL, P],
    "b200rl_upgo_head_fwd": [P, P, P, P, P, P, LL, LL, LL, P, P, P, P, c_size_t, P],
    "b200rl_upgo_head_bwd": [P, P, P, P, P, LL, LL, LL, I, P, P],
    "b200rl_vtrace_fwd": [P, P, P, P, P, P, LL, LL, LL, D, D, D, D, D, P, P, P, P, P, c_size_t, P],
    "b200rl_vtrace_continuous_fwd": [P, P, P, P, P, P, P, P, LL, LL, LL, D, D, D, D, D, P, P, P, P, P, c_size_t, P],
    "b200rl_vtrace_continuous_bwd": [P, P, P, P, P, P, P, P, P, LL, LL, LL, P, P, P, P],
    "b200rl_vtrace_fused_supported": [P, P, P, P, P, P, LL, LL, LL, P, P],
    "b200rl_vtrace_fwd_grad": [P, P, P, P, P, P, LL, LL, LL, D, D, D, D, D, P, I, P, P, P, P, P, P, P, P, P, c_size_t, P],
    "b200rl_gae_ppo_supported": [P, P, P, P, P, LL, LL, P, P, P, P, P, P, P, P, LL, P, P],
    "b200rl_gae_ppo_fwd_grad": [P, P, P, P, P, LL, LL, D, D, I, P, P, P, P, P, P, P, P, LL, D, I, D, I, P, P, P, P, P, P,
                                P, c_size_t, P],
    "b200rl_gae_ppo_fwd_grad_dp": [P, P, P, P, P, LL, LL, D, D, I, P, P, P, P, P, P, P, P, LL, D, I, D, I, P, P, P, P, P,
                                   P, P, I, I, P, P, P, c_size_t, P],
    "b200rl_p2p_drain_mean": [P, I, I, I, P, P, P],
    "b200rl_a2c_fwd_grad": [P, P, P, P, P, P, LL, LL, P, I, P, P, P, P, P, P, P, P, P, c_size_t, P],
    "b200rl_ppo_continuous_fwd_grad": [P, P, P, P, P, P, P, P, P, P, P, P, P, LL, LL, D, I, D, I, P, I, P, P, P, P, P, P, P, P, P,
                                       P, P, c_size_t, P],
    "b200rl_a2c_continuous_fwd_grad": [P, P, P, P, P, P, P, LL, LL, P, I, P, P, P, P, P, P, P, P, P, P, c_size_t, P],
    "b200rl_grpo_fwd_grad": [I, P, P, P, P, P, P, LL, LL, LL, D, D, P, P, P, P, P, c_size_t, P],
    "b200rl_rloo_fwd_grad": [I, P, P, P, P, LL, P, LL, LL, LL, D, P, P, P, P, P, c_size_t, P],
    "b200rl_token_logp_fwd": [I, P, P, LL, LL, P, P, P],
    "b200rl_token_logp_bwd": [I, P, P, P, P, P, I, LL, LL, P, P],
    "b200rl_token_head_fwd": [P, P, P, P, P, LL, P, LL, LL, D, D, P, P, P, c_size_t, P],
    "b200rl_ppo_lm_fwd_grad": [I, P, P, P, P, P, P, LL, LL, D, D, I, I, P, P, P, P, P, P, P, P, P, c_size_t, P],
    "b200rl_ppo_lm_bwd": [I, P, P, P, LL, LL, P, P, P, P, P, P, P, P, P, P, P],
    "b200rl_a2c_lm_fwd_grad": [I, P, P, P, P, P, P, LL, LL, P, P, P, P, P, P, P, P, P, P, c_size_t, P],
    "b200rl_a2c_lm_bwd": [I, P, P, P, LL, LL, P, P, P, P, P, P, P, P, P, P, P, P],
    "b200rl_gae_ppo_set_impl": [I],
    "b200rl_vtrace_set_impl": [I],
    "b200rl_acer_policy_fwd": [P, P, P, P, P, P, LL, LL, D, P, P, P],
    "b200rl_acer_policy_bwd": [P, P, P, P, P, P, P, P, LL, LL, D, P, P],
    "b200rl_acer_value_fwd": [P, P, P, LL, LL, P, P],
    "b200rl_acer_value_bwd": [P, P, P, P, LL, LL, P, P],
    "b200rl_acer_trust_region": [P, P, LL, LL, D, P, P],
    "b200rl_ppg_bc_fwd": [P, P, P, LL, LL, P, P, P, c_size_t, P],
    "b200rl_q_retraces": [P, P, P, P, P, P, LL, LL, LL, D, P, P],
    "b200rl_quantile_td_fwd": [P, P, P, P, P, P, P, P, P, LL, LL, LL, LL, LL, LL, D, LL, LL, LL, LL, LL, LL, LL, LL, I, D, P, P,
                               P, P, P, c_size_t, P],
    "b200rl_quantile_td_bwd": [P, P, P, P, P, LL, LL, LL, LL, LL, LL, I, P, P],
    "b200rl_fqf_fraction_fwd": [P, P, P, P, LL, LL, LL, LL, LL, LL, LL, LL, LL, LL, LL, LL, P, P, P, P, c_size_t, P],
    "b200rl_fqf_fraction_bwd": [P, P, LL, LL, I, P, P],
    "b200rl_p2p_allreduce_mean": [P, P, I, I, I, P, P, P],
    "b200rl_p2p_mailbox_floats": [I],
    "b200rl_probe_copy": [P, P, LL, I, P],
    "b200rl_vtrace_bwd": [P, P, P, P, P, P, P, P, LL, LL, LL, P, P, P],
}
_RESTYPE = {"b200rl_workspace_bytes": c_size_t, "b200rl_p2p_mailbox_floats": c_size_t}

_lib = None


class B200RLError(RuntimeError):
    pass


def load():
    """Load the shared library once; raise loudly if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.isfile(LIB_PATH):
        raise B200RLError(
            "di_engine_b200: CUDA library %s not found. Build it first (python __graft_entry__.py, or "
            "make -C di-engine_b200/csrc). There is no CPU fallback." % LIB_PATH
        )
    lib = ctypes.CDLL(LIB_PATH)
    for name, argtypes in PROTOTYPES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.argtypes = argtypes
        fn.restype = _RESTYPE.get(name, c_int)
    _lib = lib
    return lib


def check(rc, what):
    if rc == 0:
        return
    if rc == -1:
        raise B200RLError("%s: invalid argument (B200RL_ERR_ARG)" % what)
    if rc == -2:
        raise B200RLError("%s: workspace too small for this problem size (B200RL_ERR_WORKSPACE)" % what)
    raise B200RLError("%s: CUDA error %d at launch" % (what, rc))
