"""Value rescaling helpers h / h^-1 (ding/rl_utils/value_rescale.py:4-34) and symlog / inv_symlog (:37-66).

Inside ``q_nstep_td_error_with_rescale`` the default pair h / h^-1 is evaluated in the fused CUDA kernel (csrc/td.cu
``value_h`` / ``value_h_inv``); these tensor-level versions exist because they are the default ``trans_fn`` /
``inv_trans_fn`` arguments of that signature and part of the public namespace.  ``symlog`` / ``inv_symlog`` are
PPOFPolicy's value normalisation (ding/policy/ppof.py:185-186, :203-204) and run on csrc/policy.cu's element-wise kernel,
forward and backward.
"""
import torch

from .. import ops, torch_ops


def value_transform(x: torch.Tensor, eps: float = 1e-2) -> torch.Tensor:
    """h(x) = sign(x)(sqrt(|x|+1) - 1) + eps*x  (arXiv:1805.11593)."""
    root = torch.sqrt(x.abs() + 1) - 1
    return x.sign() * root + eps * x


def value_inv_transform(x: torch.Tensor, eps: float = 1e-2) -> torch.Tensor:
    """h^-1(x) = sign(x)(((sqrt(1 + 4 eps (|x| + 1 + eps)) - 1) / (2 eps))^2 - 1)."""
    inner = torch.sqrt(1 + 4 * eps * (x.abs() + 1 + eps))
    return x.sign() * (((inner - 1) / (2 * eps)) ** 2 - 1)


def _value_map(x, mode, name):
    if not isinstance(x, torch.Tensor) or x.dtype != torch.float32:
        raise TypeError("di_engine_b200: %s takes a float32 tensor (got %s); the CUDA path computes in fp32" %
                        (name, getattr(x, 'dtype', type(x).__name__)))
    dev = ops.compute_device(x)
    xd = ops.to_device(x, dev).contiguous()
    y = torch_ops.value_map(xd, mode) if torch.compiler.is_compiling() else ops.ValueMapFunction.apply(xd, mode)
    return y if x.is_cuda else y.cpu()


def symlog(x: torch.Tensor) -> torch.Tensor:
    """symlog(x) = sign(x) * log(|x| + 1)  (arXiv:2301.04104), differentiable.  fp32 only: other dtypes raise TypeError.
    A host tensor is computed on the current CUDA device and the result returned on the host."""
    return _value_map(x, 0, 'symlog')


def inv_symlog(x: torch.Tensor) -> torch.Tensor:
    """symexp(x) = sign(x) * (exp(|x|) - 1), the inverse of ``symlog``, differentiable.  fp32 only, as ``symlog``."""
    return _value_map(x, 1, 'inv_symlog')
