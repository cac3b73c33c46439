"""Mirror of the hot-path part of ``ding.rl_utils`` (ding/rl_utils/__init__.py:1-27): identical names, signatures and
namedtuples, computed by the sm_90a kernels behind the C ABI of ``include/b200rl.h``."""
from .a2c import a2c_data, a2c_error, a2c_error_continuous, a2c_loss
from .acer import acer_policy_error, acer_trust_region_update, acer_value_error
from .coma import coma_data, coma_error, coma_loss
from .fused import gae_ppo_error
from .happo import (happo_data, happo_error, happo_error_continuous, happo_policy_error_continuous, happo_info, happo_loss, happo_policy_data, happo_policy_error, happo_policy_loss,
                    happo_value_data, happo_value_error)
from .grpo import grpo_info, grpo_policy_data, grpo_policy_error
from .log_prob_utils import efficient_method, less_efficient_method, naive_method
# composites from the lm_head's hidden states (not reference names: outside the hot-path lists below)
from .lm_linear import (a2c_error_linear, a2c_linear_data, a2c_linear_loss, grpo_linear_data, grpo_policy_error_linear,
                        ppo_linear_loss, ppo_policy_error_linear, ppo_policy_linear_data, rloo_linear_data,
                        rloo_policy_error_linear, token_logp_linear)
from .gae import gae, gae_data, gae_returns, gae_returns_out, ppof_gae_returns, ppof_gae_returns_out, shape_fn_gae
from .ppo import (normalize_advantage, ppo_data, ppo_data_continuous, ppo_error, ppo_error_adv_norm, ppo_error_continuous, ppo_info, ppo_loss,
                  ppo_policy_data, ppo_policy_data_continuous, ppo_policy_error, ppo_policy_error_continuous, ppo_policy_loss,
                  ppo_value_data, ppo_value_error, shape_fn_ppo)
from .td import (bdq_nstep_td_error, dist_1step_td_data, dist_1step_td_error, dist_nstep_td_data, dist_nstep_td_error,
                 dqfd_nstep_td_data, dqfd_nstep_td_error, dqfd_nstep_td_error_sequence, dqfd_nstep_td_error_with_rescale,
                 dqfd_nstep_td_seq_data, generalized_lambda_returns, m_q_1step_td_data, m_q_1step_td_error, q_1step_td_data,
                 q_1step_td_error, q_nstep_sql_td_error, q_nstep_td_data, q_nstep_td_error, q_nstep_td_error_sequence,
                 q_nstep_td_error_with_rescale, q_nstep_td_seq_data, q_v_1step_td_data, q_v_1step_td_error, shape_fn_dntd,
                 shape_fn_qntd, shape_fn_qntd_rescale, shape_fn_td_lambda, td_lambda_data, td_lambda_error,
                 v_1step_td_data, v_1step_td_error, v_nstep_td_data, v_nstep_td_error)
from .ppg import ppg_data, ppg_joint_error, ppg_joint_loss
from .quantile import (fqf_calculate_fraction_loss, fqf_nstep_td_data, fqf_nstep_td_error, iqn_nstep_td_data,
                       iqn_nstep_td_error, qrdqn_nstep_td_data, qrdqn_nstep_td_error)
from .retrace import compute_q_retraces
from .rloo import rloo_info, rloo_policy_data, rloo_policy_error
from .upgo import tb_cross_entropy, upgo_loss, upgo_returns
from .value_rescale import inv_symlog, symlog, value_inv_transform, value_transform
from .vtrace import (impala_reshape_data, shape_fn_vtrace_discrete_action, vtrace_data, vtrace_error_continuous_action,
                     vtrace_error_discrete_action, vtrace_loss)

HOT_PATH_FUNCTIONS = [
    'gae', 'ppo_error', 'q_nstep_td_error', 'q_nstep_td_error_with_rescale', 'dist_nstep_td_error', 'td_lambda_error',
    'generalized_lambda_returns', 'upgo_loss', 'vtrace_error_discrete_action',
    # siblings on the same kernels (SURVEY section 8f)
    'q_1step_td_error', 'v_1step_td_error', 'v_nstep_td_error', 'ppo_policy_error', 'ppo_value_error',
    'dist_1step_td_error', 'bdq_nstep_td_error', 'upgo_returns', 'tb_cross_entropy', 'ppo_error_continuous', 'a2c_error',
    'vtrace_error_continuous_action', 'qrdqn_nstep_td_error', 'iqn_nstep_td_error', 'fqf_nstep_td_error',
    'fqf_calculate_fraction_loss', 'compute_q_retraces', 'happo_error', 'happo_policy_error', 'happo_value_error', 'happo_error_continuous', 'happo_policy_error_continuous',
    'acer_policy_error', 'acer_value_error', 'acer_trust_region_update', 'ppg_joint_error',
    'dqfd_nstep_td_error', 'dqfd_nstep_td_error_with_rescale',
    'm_q_1step_td_error', 'q_nstep_sql_td_error', 'q_v_1step_td_error',
    'a2c_error_continuous', 'ppo_policy_error_continuous',
    # PPOFPolicy's value normalisation (ding/policy/ppof.py:13)
    'symlog', 'inv_symlog'
]
HOT_PATH_TYPES = [
    'gae_data', 'ppo_data', 'ppo_loss', 'ppo_info', 'q_nstep_td_data', 'dist_nstep_td_data', 'td_lambda_data',
    'vtrace_data', 'vtrace_loss', 'q_1step_td_data', 'v_1step_td_data', 'v_nstep_td_data',
    'ppo_policy_data', 'ppo_policy_loss', 'ppo_value_data', 'dist_1step_td_data', 'a2c_data', 'a2c_loss',
    'qrdqn_nstep_td_data', 'iqn_nstep_td_data', 'fqf_nstep_td_data',
    'happo_data', 'happo_policy_data', 'happo_value_data', 'happo_loss', 'happo_policy_loss', 'happo_info', 'ppg_data', 'ppg_joint_loss',
    'dqfd_nstep_td_data', 'm_q_1step_td_data', 'q_v_1step_td_data', 'ppo_data_continuous', 'ppo_policy_data_continuous'
]
# the language-model losses (ding/rl_utils/{grpo,rloo,log_prob_utils}.py), listed apart from the classic hot path above:
# the test suite's reference loader covers only the files those lists come from.  install() rebinds both lists
LM_HOT_PATH_FUNCTIONS = [
    'grpo_policy_error', 'rloo_policy_error', 'naive_method', 'efficient_method', 'less_efficient_method'
]
LM_HOT_PATH_TYPES = ['grpo_policy_data', 'grpo_info', 'rloo_policy_data', 'rloo_info']
# COMA (ding/rl_utils/coma.py), listed apart for the same reason; install() rebinds it with the lists above
COMA_HOT_PATH_FUNCTIONS = ['coma_error']
