"""``upgo_loss`` / ``upgo_returns`` / ``tb_cross_entropy`` with the signatures of ding/rl_utils/upgo.py:7,46,77 -- csrc/td.cu +
csrc/pg.cu."""
import torch

from .. import ops, torch_ops


def tb_cross_entropy(logit: torch.Tensor, label: torch.Tensor, mask=None) -> torch.Tensor:
    """
    Time-batch cross entropy "with the sign of a log-probability", drop-in for ding/rl_utils/upgo.py:7-43:
    ``-F.cross_entropy(logit, label)`` per (t, b); logit (T, B, N) with label (T, B), or (T, B, N2, N) with label / mask
    (T, B, N2), the masked per-entry values summed over N2 (the mask is ignored for 3-D logits, as in the reference).
    Returns (T, B), differentiable w.r.t. ``logit``.
    """
    assert (len(label.shape) >= 2)  # upgo.py:23
    T, B = label.shape[:2]
    K = 1
    if len(label.shape) > 2:
        assert len(label.shape) == 3  # upgo.py:27
        K = label.shape[2]
    N = logit.shape[-1]
    dev = ops.compute_device(logit)
    host_out = not logit.is_cuda
    if logit.numel() != T * B * K * N:
        raise ValueError("logit %s does not match label %s" % (tuple(logit.shape), tuple(label.shape)))
    z = ops.f32c(ops.to_device(logit, dev), 'logit')
    lab = ops.i64c(ops.to_device(label, dev), logit.shape[-1], 'label')
    m = None
    if mask is not None and K > 1:
        m = ops.f32c(ops.to_device(mask.detach(), dev), 'mask')
    ce = ops.TBCrossEntropyFunction.apply(z, lab, m, T * B, K, N).reshape(T, B)
    return ce.cpu() if host_out else ce


def upgo_returns(rewards: torch.Tensor, bootstrap_values: torch.Tensor) -> torch.Tensor:
    """
    UPGO return targets (ding/rl_utils/upgo.py:46-68): a lambda-return with gamma = 1 whose trace continues
    (lambda_t = 1) while r_{t+1} + V_{t+2} >= V_{t+1}.  rewards (T, B), bootstrap_values (T+1, B) -> (T, B).
    The comparison and the recurrence are evaluated in one kernel, bit-exact with the reference; as in the reference the
    result is differentiable w.r.t. both inputs (no gradient flows through the comparison).
    """
    dev = ops.compute_device(rewards, bootstrap_values)
    host_out = not rewards.is_cuda
    grad_on = torch.is_grad_enabled()
    rg_v, rg_r = bootstrap_values.requires_grad and grad_on, rewards.requires_grad and grad_on
    v = ops.f32c(ops.to_device(bootstrap_values if rg_v else bootstrap_values.detach(), dev), 'bootstrap_values')
    r = ops.f32c(ops.to_device(rewards if rg_r else rewards.detach(), dev), 'rewards')
    if rg_v or rg_r:
        ret = ops.LambdaReturnsFunction.apply(v, r, None, None, None, 1.0, 1.0, True)
    else:
        ret = ops.lambda_returns_(v, r, None, 1.0, None, 1.0, None, True)
    return ret.cpu() if host_out else ret


def upgo_loss(
        target_output: torch.Tensor,
        rhos: torch.Tensor,
        action: torch.Tensor,
        rewards: torch.Tensor,
        bootstrap_values: torch.Tensor,
        mask=None
) -> torch.Tensor:
    """
    Importance-weighted UPGO policy-gradient loss, drop-in for ding/rl_utils/upgo.py:77-111.
    target_output (T, B, N) with action (T, B) -- or (T, B, N2, N) with action / mask (T, B, N2) (upgo.py:25-37);
    rhos, rewards (T, B); bootstrap_values (T+1, B).  Gradient reaches ``target_output`` only.
    """
    dev = ops.compute_device(target_output, rewards)
    host_out = not target_output.is_cuda
    assert action.dim() >= 2  # upgo.py:23
    T, B = action.shape[:2]
    N = target_output.shape[-1]
    if action.dim() > 2:
        assert action.dim() == 3  # upgo.py:27
        K = action.shape[2]
    else:
        K = 1
    if target_output.numel() != T * B * K * N:
        raise ValueError("target_output %s does not match action %s" % (tuple(target_output.shape),
                                                                        tuple(action.shape)))
    logit = ops.f32c(ops.to_device(target_output, dev), 'target_output')
    act = ops.i64c(ops.to_device(action, dev), target_output.shape[-1])
    m = None
    if mask is not None and K > 1:  # the reference ignores mask for 3-D logits (upgo.py:38-42)
        m = ops.f32c(ops.to_device(mask.detach(), dev), 'mask')
    rho = ops.f32c(ops.to_device(rhos.detach(), dev), 'rhos')
    r = ops.f32c(ops.to_device(rewards.detach(), dev), 'rewards')
    v = ops.f32c(ops.to_device(bootstrap_values.detach(), dev), 'bootstrap_values')
    if torch.compiler.is_compiling():
        loss = torch_ops.upgo(logit, act, m, rho, r, v, T * B, K, N)
    else:
        ret = ops.lambda_returns_(v, r, None, 1.0, None, 1.0, None, True)
        loss = ops.UPGOFunction.apply(logit, act, m, rho, ret, v, T * B, K, N)
    return loss.cpu() if host_out else loss
