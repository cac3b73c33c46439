"""TEST INFRASTRUCTURE ONLY -- float64 restatement of COMA's loss, ``coma_error`` (ding/rl_utils/coma.py:10-58), in numpy,
with its gradients written out.  The product package never imports it.

    q_t = q_value[.., action], v_t = target_q_value[.., action], r_t = reward[t, b] for every agent a
    G_{T-2} = r_{T-2} + gamma v_{T-1};  G_t = r_t + gamma (lambda G_{t+1} + (1 - lambda) v_{t+1})        (td.py:1574-1651)
    q_value_loss = mean_{t<T-1} w (G - q)^2                       policy_loss = -mean logp(action) adv w
    adv = q - sum_j softmax(logit)_j q_value_j (detached)         entropy_loss = mean H w,  H = -sum_j p_j max(logp_j, fp32 min)
"""
import numpy as np

F32_MIN = float(np.finfo(np.float32).min)


def coma(logit, action, q_value, target_q_value, reward, weight, gamma, lambda_, upstream=(1.0, 1.0, 1.0)):
    """-> dict of the three losses and d (upstream . losses) / d logit, q_value, target_q_value, reward, float64"""
    z = np.asarray(logit, np.float64)
    q = np.asarray(q_value, np.float64)
    tq = np.asarray(target_q_value, np.float64)
    act = np.asarray(action, np.int64)
    T, B, A, N = z.shape
    w = np.ones((T, B, A)) if weight is None else np.broadcast_to(np.asarray(weight, np.float64), (T, B, A))
    r = np.broadcast_to(np.asarray(reward, np.float64)[:, :, None], (T, B, A))
    take = lambda x: np.take_along_axis(x, act[..., None], -1)[..., 0]  # noqa: E731
    qt, vt = take(q), take(tq)
    G = np.empty((T - 1, B, A))
    G[-1] = r[T - 2] + gamma * vt[T - 1]
    for t in range(T - 3, -1, -1):
        G[t] = r[t] + gamma * (lambda_ * G[t + 1] + (1 - lambda_) * vt[t + 1])
    d = G - qt[:-1]
    M, R = (T - 1) * B * A, T * B * A
    value_loss = (w[:-1] * d * d).sum() / M
    with np.errstate(invalid='ignore', divide='ignore', over='ignore'):
        m = z.max(-1, keepdims=True)
        lp = (z - m) - np.log(np.exp(z - m).sum(-1, keepdims=True))
        p = np.exp(lp)
        lpc = np.maximum(lp, F32_MIN)
        ent = -(p * lpc).sum(-1)
        adv = qt - (p * q).sum(-1)
        lpa = take(lp)
        policy_loss = -(lpa * adv * w).sum() / R
        entropy_loss = (ent * w).sum() / R
        u0, u1, u2 = upstream
        onehot = np.zeros_like(z)
        np.put_along_axis(onehot, act[..., None], 1.0, -1)
        g_logit = (u0 * (-adv * w / R))[..., None] * (onehot - p) + (u2 * w / R)[..., None] * (-p * (lpc + ent[..., None]))
    g_q = np.zeros_like(q)
    np.put_along_axis(g_q[:-1], act[:-1, ..., None], (u1 * -2 * w[:-1] * d / M)[..., None], -1)
    dG = u1 * 2 * w[:-1] * d / M
    a = np.zeros((B, A))
    g_v = np.zeros((T, B, A))
    g_r = np.zeros((T, B))
    for t in range(T - 1):  # the transposed recurrence runs forward in time
        a = dG[t] + (gamma * lambda_ * a if t > 0 else 0.0)
        g_r[t] = a.sum(-1)
        g_v[t + 1] = a * (gamma if t == T - 2 else gamma * (1 - lambda_))
    g_tq = np.zeros_like(tq)
    np.put_along_axis(g_tq, act[..., None], g_v[..., None], -1)
    return {'policy_loss': policy_loss, 'q_value_loss': value_loss, 'entropy_loss': entropy_loss, 'grad_logit': g_logit,
            'grad_q_value': g_q, 'grad_target_q_value': g_tq, 'grad_reward': g_r}
