"""TEST INFRASTRUCTURE ONLY -- float64 restatement of FQF's fraction loss, ``fqf_calculate_fraction_loss``
(ding/rl_utils/td.py:1485-1511), in numpy.  The product package never imports it.

    s_i  = q_tau_i[b, i, a_b]  (i < N-1)          h_k = q_value[b, k, a_b]  (k < N)
    g_i  = where(s_i > (i == 0 ? h_0 : s_{i-1}), s_i - h_i, -(s_i - h_i))
         + where(s_i < (i == N-2 ? h_{N-1} : s_{i+1}), s_i - h_{i+1}, -(s_i - h_{i+1}))
    loss = mean_b sum_i g_i * quantiles[b, i+1]
    d loss / d quantiles[b, i+1] = u / B * g_i,   columns 0 and N: 0

A comparison with NaN is false, so a NaN operand takes the negated branch (NaN either way).
"""
import numpy as np


def fraction_terms(q_tau_i, q_value, actions):
    """-> g (B, N-1), float64"""
    act = np.asarray(actions, np.int64)[:, None, None]
    s = np.take_along_axis(np.asarray(q_tau_i), act, 2)[:, :, 0].astype(np.float64)  # (B, N-1)
    h = np.take_along_axis(np.asarray(q_value), act, 2)[:, :, 0].astype(np.float64)  # (B, N)
    lo = np.concatenate([h[:, :1], s[:, :-1]], 1)  # the left neighbour of s_i: h_0 for i = 0
    hi = np.concatenate([s[:, 1:], h[:, -1:]], 1)  # the right neighbour: h_{N-1} for i = N-2
    v1, v2 = s - h[:, :-1], s - h[:, 1:]
    with np.errstate(invalid='ignore'):
        return np.where(s > lo, v1, -v1) + np.where(s < hi, v2, -v2)


def fraction_loss(q_tau_i, q_value, quantiles, actions, upstream=1.0):
    """-> (loss, d (upstream * loss) / d quantiles (B, N+1)), float64"""
    g = fraction_terms(q_tau_i, q_value, actions)
    qn = np.asarray(quantiles, np.float64)
    B = g.shape[0]
    with np.errstate(invalid='ignore'):
        loss = float((g * qn[:, 1:-1]).sum(1).mean())
        grad = np.zeros_like(qn)
        grad[:, 1:-1] = upstream / B * g
    return loss, grad
