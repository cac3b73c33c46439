"""The one-launch GAE + ppo_error step on the column-tile kernel (csrc/colws.cu) at the shapes where it picks its
32-column geometry on an H100 (132 SMs: B from 3940 to 4224), and at their ragged neighbours: B not a multiple of 32, T
not a multiple of the 8-step chunk, N from 1 to 21, with and without logit_pretrained / weight.  Checked against the
oracle with the tolerances of test_gpu_parity.test_fused_gae_ppo_matches_oracle (advantages bit-identical)."""
import pytest

from di_engine_b200 import _lib
from tests.test_gpu_parity import _fused_vs_oracle


@pytest.fixture
def col_impl():
    lib = _lib.load()
    old = lib.b200rl_gae_ppo_set_impl(2)
    yield
    lib.b200rl_gae_ppo_set_impl(old)


@pytest.mark.gpu
@pytest.mark.parametrize('T, B, N', [(128, 4096, 6), (131, 4096, 6), (125, 4100, 6), (128, 4100, 1), (128, 4096, 18),
                                     (67, 4068, 21), (9, 4224, 6), (3, 3972, 6)])
def test_colws_wide_matches_oracle(T, B, N, col_impl):
    _fused_vs_oracle(T, B, N, seed=900 + T + N)


@pytest.mark.gpu
@pytest.mark.parametrize('T, B, N, weight, pretrained', [(128, 4096, 6, 'tensor', False), (61, 4100, 6, 'none', True),
                                                          (128, 4096, 21, 'tensor', False), (36, 4100, 1, 'tensor', True),
                                                          (40, 4096, 14, 'none', True)])
def test_colws_wide_weight_pretrained(T, B, N, weight, pretrained, col_impl):
    mix = (1.0, 0.5, -0.01, 0.2 if pretrained else 0.0)
    _fused_vs_oracle(T, B, N, seed=950 + T + N, weight=weight, pretrained=pretrained, mix=mix,
                     kl_type='k3' if pretrained else 'k1')


@pytest.mark.gpu
def test_colws_wide_forward_only(col_impl):
    _fused_vs_oracle(128, 4100, 6, 990, grad=False)


def test_gae_ppo_supported_every_n_at_config_d():
    """b200rl_gae_ppo_supported is host arithmetic on shapes and addresses: at T = 128, B = 4096 every N from 1 to 32,
    with and without logit_pretrained and weight, has a one-launch kernel"""
    lib = _lib.load()
    a = 1 << 20  # any 16-byte aligned address: nothing is dereferenced
    for N in range(1, 33):
        for pre in (None, a):
            for w in (None, a):
                assert lib.b200rl_gae_ppo_supported(a, a, a, a, a, 128, 4096, a, a, pre, a, a, a, a, w, N, a, a) == 1, \
                    (N, pre, w)
